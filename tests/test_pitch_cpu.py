"""Pitch and gain without a GPU: the request's mapping (rho, q, g) and its refusals, the C and Python twins of the
resampler at a pitch (constants, counts, design), the float64 oracle at a pitch against scipy, the pitch it moves a sine
to, and the plumbing of every generate method, the batcher and the server."""
import ctypes as C
import importlib.util
import inspect
import math
import os
import re
import types

import numpy as np
import pytest
import torch

from oracle import prompt_cases  # noqa: F401  (puts the package on sys.path)
from oracle import resample_oracle as RO
from oracle import tempo_oracle as TO
import pitch_oracle as P
from faster_qwen3_tts import resample as R
from faster_qwen3_tts import tempo as T
from faster_qwen3_tts.model import FasterQwen3TTS, _post_kw
from faster_qwen3_tts.serving import ContinuousBatcher

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BAD_PITCH = (12.01, -12.5, 24, float("nan"), float("inf"), "1", None, True)
BAD_GAIN = (-96.01, 16.5, 100, float("nan"), -float("inf"), "0", None, False)
# (speed, pitch) pairs whose tempo leaves [256, 4096]: just past the corners of the admitted range
BAD_COMBOS = ((0.25, 0.1), (4.0, -0.1), (0.498, 12), (2.01, -12), (0.3, 4), (3.0, -7))


def test_rho_q_and_gain_mapping():
    assert [R.pitch_rho(p) for p in (-12, -7, -5, 0, 4, 7, 12)] == [128, 171, 192, 256, 323, 384, 512]
    for p in np.linspace(-12, 12, 241):
        rho = R.pitch_rho(p)
        assert rho == P.rho_of(p) and 128 <= rho <= 512
        assert abs(1200 * math.log2(rho / 256) - 100 * p) <= 6.76   # cents off the request: half a step of 1/128 at rho 128
    # the corners: every speed in [0.5, 2] meets every pitch in [-12, 12]
    assert R.tempo_q(0.5, 12) == 256 and R.tempo_q(2, -12) == 4096 and R.tempo_q(2, 12) == 1024
    assert R.tempo_q(0.5, -12) == 1024 and R.tempo_q(1.5, 7) == 1024   # tape speed: no tempo
    for s in np.linspace(0.5, 2, 61):
        for p in np.linspace(-12, 12, 25):
            assert 256 <= R.tempo_q(s, p) <= 4096
    # at pitch 0 q is the plain speed's, bit for bit, ties included
    for s in list(np.linspace(0.25, 4, 397)) + [1 + 1 / 2048, 1 - 1 / 2048, 1.0004, 0.25, 4.0]:
        assert R.tempo_q(s, 0) == T.quantize(s) == P.tempo_q(s, 0)
        assert R.tempo_speed(s, 0) is s
    assert R.tempo_speed(1.0, 7) == 683 / 1024 and T.quantize(R.tempo_speed(1.0, 7)) == 683
    assert R.gain_of(0) == 1.0 and R.gain_of(-0.0) == 1.0
    for db in (-96, -6, -0.5, 3, 16):
        assert R.gain_of(db) == float(np.float32(10 ** (db / 20))) == float(P.gain_of(db))
    assert R.check_prosody(1.0, 0, 0) == (1024, 256, 1.0)


@pytest.mark.parametrize("speed,pitch", BAD_COMBOS)
def test_impossible_speed_and_pitch_are_refused_naming_both(speed, pitch):
    with pytest.raises(ValueError) as e:
        R.check_prosody(speed, pitch, 0)
    assert f"speed {speed!r}" in str(e.value) and f"pitch {pitch!r}" in str(e.value)


def test_out_of_range_values_are_refused():
    for p in BAD_PITCH:
        with pytest.raises(ValueError, match="pitch"):
            R.check_prosody(1.0, p, 0)
    for g in BAD_GAIN:
        with pytest.raises(ValueError, match="gain_db"):
            R.check_prosody(1.0, 0, g)
    with pytest.raises(ValueError, match="speed"):
        R.check_prosody(5.0, 12, 0)   # the speed's own range still holds


def test_constants_agree_with_the_c_header():
    h = open(os.path.join(ROOT, "include", "fq3_engine.h")).read()
    val = dict(re.findall(r"#define FQ3_RESAMPLE_(\w+) ([0-9.]+)", h))
    assert (int(val["PITCH_ONE"]), int(val["PITCH_MIN"]), int(val["PITCH_MAX"])) == (R.PITCH_ONE, R.PITCH_MIN,
                                                                                     R.PITCH_MAX)
    assert int(val["TABLE_CACHE"]) == R.TABLE_CACHE
    assert (R.pitch_rho(-12), R.pitch_rho(12)) == (R.PITCH_MIN, R.PITCH_MAX)


def test_plain_rates_are_unchanged():
    """at rho 256 the ratios, counts and the oracle are the plain rate's exactly"""
    rng = np.random.default_rng(0)
    x = rng.standard_normal(700)
    for rate in R.RATES:
        assert R.ratio(rate, 256) == R.ratio(rate) == RO.ratio(rate) == P.ratio(rate, 256)
        assert np.array_equal(P.design(rate, 256), RO.design(rate))
        assert np.array_equal(P.resample(x, rate, 256), RO.resample(x, rate))
        for t in (0, 1, 99, 1234):
            for f in (False, True):
                assert R.emitted(t, rate, f, 256) == R.emitted(t, rate, f)


def _pitched_cases():
    rng = np.random.default_rng(7)
    cases = [(22050, 509), (44100, 509), (8000, 512), (48000, 128), (24000, 383), (16000, 181), (48000, 512)]
    cases += [(int(rng.choice(R.RATES)), int(rng.integers(128, 513))) for _ in range(6)]
    return cases


def _lib():
    from faster_qwen3_tts.engine import LIB_PATH, load_library
    if not os.path.exists(LIB_PATH):
        pytest.skip("the extension is not built")
    return load_library()


@pytest.mark.parametrize("rate,rho", _pitched_cases())
def test_c_and_python_twins_agree(rate, rho):
    """fq3_resample_taps_pitch / fq3_resample_released_pitch against the oracle's design and resample.py's counts"""
    lib = _lib()
    L, M, half = R.ratio(rate, rho)
    assert (L, M, half) == P.ratio(rate, rho)
    n = lib.fq3_resample_taps_pitch(rate, rho, None, 0)
    assert n == 2 * half + 1
    buf = (C.c_double * n)()
    assert lib.fq3_resample_taps_pitch(rate, rho, buf, n) == n
    assert np.abs(np.frombuffer(buf, dtype=np.float64) - P.design(rate, rho)).max() <= 1e-14
    rng = np.random.default_rng(rate + rho)
    for _ in range(2000):
        t, m, f = int(rng.integers(0, 10 ** 6)), int(rng.integers(0, 20000)), bool(rng.integers(0, 2))
        assert lib.fq3_resample_released_pitch(rate, rho, t, m, int(f)) == R.released(t, m, rate, f, rho)
    for t in range(100):
        for m in range(3):
            assert lib.fq3_resample_released_pitch(rate, rho, t, m, 0) == R.released(t, m, rate, False, rho)
    assert lib.fq3_resample_released_pitch(rate, 127, 0, 1, 0) == -1
    assert lib.fq3_resample_taps_pitch(rate, 513, None, 0) == -1


def test_largest_tables():
    """22.05 and 44.1 kHz at rho 509 are the largest designs: 162 881 taps, about 0.65 MB of table"""
    signal = pytest.importorskip("scipy.signal")
    for rate in (22050, 44100):
        L, M, half = R.ratio(rate, 509)
        assert 2 * half + 1 == 162881
        assert L * (2 * half // L + 1) * 4 <= 660_000
        want = signal.firwin(2 * half + 1, 0.9 / max(L, M), window=("kaiser", 8.6))
        assert np.abs(P.design(rate, 509) - want).max() <= 1e-15
    sizes = [R.ratio(r, rho) for r in R.RATES for rho in range(128, 513)]
    assert max(2 * h // L + 1 for L, M, h in sizes) == 385                       # taps per output (8 kHz, rho 512)
    assert max(-(-2 * h // L) for L, M, h in sizes) == 384                       # tail samples


@pytest.mark.parametrize("rate,rho", [(8000, 171), (16000, 384), (24000, 192), (48000, 323), (32000, 509),
                                      (22050, 256), (44100, 181)])
def test_oracle_design_is_firwin_and_output_is_resample_poly(rate, rho):
    signal = pytest.importorskip("scipy.signal")
    L, M, half = P.ratio(rate, rho)
    h = P.design(rate, rho)
    want = signal.firwin(2 * half + 1, 0.9 / max(L, M), window=("kaiser", 8.6))
    assert np.abs(h - want).max() <= 1e-15
    rng = np.random.default_rng(rate + rho)
    for n in (1, 37, 1500):
        x = rng.standard_normal(n)
        y = P.resample(x, rate, rho)
        ref = signal.resample_poly(x, L, M, window=h)
        assert len(y) == len(ref) == -(-n * L // M)
        assert np.abs(y - ref).max() <= 1e-12


@pytest.mark.parametrize("rate,rho", [(8000, 512), (44100, 181), (24000, 383), (16000, 128)])
def test_oracle_counts_and_chunking_invariance(rate, rho):
    rng = np.random.default_rng(rate * rho)
    x = rng.standard_normal(900)
    whole = P.resample(x, rate, rho)
    st, parts, tot, i = P.Stream(rate, rho), [], 0, 0
    while i < len(x):
        n = min(int(rng.integers(0, 200)), len(x) - i)
        fin = i + n == len(x)
        r = st.push(x[i:i + n], fin)
        assert len(r) == R.released(tot, n, rate, fin, rho)
        parts.append(r)
        tot, i = tot + n, i + n
    assert np.allclose(np.concatenate(parts), whole, rtol=0, atol=0)


@pytest.mark.parametrize("rate,pitch,speed", [(24000, 7, 1.0), (8000, -5, 1.0), (48000, 4, 1.5), (16000, -12, 1.0),
                                              (24000, 12, 0.75)])
def test_tempo_then_resample_moves_a_sine_to_its_pitch(rate, pitch, speed):
    """on the oracles: a 24 kHz sine at f, stretched at q and resampled at (R, rho), peaks at f rho / 256 (within an
    FFT bin), and lasts the closed-form count"""
    rho, q = R.pitch_rho(pitch), R.tempo_q(speed, pitch)
    f = 440.0 if rho > 256 else 1000.0
    n = 24000
    x = 0.5 * np.sin(2 * np.pi * f * np.arange(n) / 24000)
    y, _ = TO.stretch(x, q / 1024)
    assert len(y) == T.out_len(n, q)
    z = P.resample(y, rate, rho)
    L, M, _ = R.ratio(rate, rho)
    assert len(z) == -(-T.out_len(n, q) * L // M) == R.released(0, len(y), rate, True, rho)
    w = z[len(z) // 8: len(z) - len(z) // 8]
    spec = np.abs(np.fft.rfft(w * np.hanning(len(w))))
    peak = np.argmax(spec) * rate / len(w)
    assert abs(peak - f * rho / 256) <= rate / len(w), (peak, f * rho / 256)
    assert abs(len(z) / rate - (n / 24000) * 2 ** 18 / (q * rho)) <= 2 / rate
    assert abs(2 ** 18 / (q * rho) * speed - 1) < 0.002


def test_post_kw_at_pitch_zero_and_zero_db_is_today_s():
    for speed in (1.0, 1.5, 0.25):
        for rate in (None, 24000, 8000, 48000):
            want = {} if speed == 1.0 else {"speed": speed}
            if rate is not None and rate != 24000:
                want["sample_rate"] = rate
            assert _post_kw(speed, rate) == _post_kw(speed, rate, 0, 0) == _post_kw(speed, rate, 0.0, -0.0) == want
    assert _post_kw(1.0, None, 3, 0) == {"pitch": 3} and _post_kw(1.0, None, 0, -6) == {"gain_db": -6}


def test_identity_creates_nothing():
    assert R.resampler_for(None, "f32", None, 0, 0) is None and R.resampler_for(24000, "f32", None, 0.0, -0.0) is None
    R.warm(24000, "f32", "cpu", 0)   # pitch 0: nothing to design


def _boom_model():
    class Boom:
        def __getattr__(self, name):
            raise AssertionError(f"touched the model ({name}) before pitch / gain were checked")

    m = FasterQwen3TTS.__new__(FasterQwen3TTS)
    m.model = Boom()
    return m


def test_every_generate_method_takes_pitch_and_gain_and_refuses_before_tokenizing():
    m = _boom_model()
    names = [n for n in dir(FasterQwen3TTS) if n.startswith("generate_")] + ["stream_from_embeds",
                                                                              "stream_batch_from_embeds"]
    assert len(names) == 15
    for name in names:
        p = inspect.signature(getattr(FasterQwen3TTS, name)).parameters
        assert p["pitch"].default == 0 and p["gain_db"].default == 0, name
        keys = list(p)
        assert keys[keys.index("sample_rate") + 1:keys.index("sample_rate") + 3] == ["pitch", "gain_db"], name
        batch = name == "generate_custom_voice_batch"
        args = [["x"] if batch else "x" for k, v in p.items() if k != "self" and v.default is inspect.Parameter.empty]
        bad = [dict(pitch=p_) for p_ in (13, float("nan"))] + [dict(gain_db=g) for g in (17, float("inf"))] + \
            [dict(speed=s, pitch=p_) for s, p_ in BAD_COMBOS[:2]]
        for kw in bad:
            with pytest.raises(ValueError):
                r = getattr(m, name)(*args, **kw)
                if inspect.isgenerator(r):
                    next(r)


def test_text_streaming_takes_pitch_and_gain():
    from faster_qwen3_tts.text_stream import generate_text_streaming
    p = inspect.signature(generate_text_streaming).parameters
    assert p["pitch"].default == 0 and p["gain_db"].default == 0


# ---- ContinuousBatcher and the server, on fakes -------------------------------------------------------------------
class _Sched:
    def has_capacity(self):
        return True

    def submit(self, tie, tam, tth, tpe, tag, **kw):
        return types.SimpleNamespace(tag=tag, finished=0, done=0, due=0.0, hold=False)

    def cancel(self, rq):
        pass

    def __len__(self):
        return 0

    def step(self, chunk):
        return []


def _batcher():
    calls, warmed = [], []

    def window(ref_codes, **kw):
        calls.append(kw)
        raise RuntimeError("not run")
    window.warm = lambda *a: warmed.append(a)
    return ContinuousBatcher(_Sched(), window, chunk_size=8, sleep=lambda s: None), calls, warmed


def test_submit_refuses_bad_pitch_gain_and_combinations():
    b, calls, warmed = _batcher()
    try:
        for kw in [dict(pitch=p) for p in BAD_PITCH] + [dict(gain_db=g) for g in BAD_GAIN] + \
                [dict(speed=s, pitch=p) for s, p in BAD_COMBOS]:
            with pytest.raises(ValueError):
                b.submit(lambda: None, **kw)
            b.feed_factory = lambda n: None
            with pytest.raises(ValueError):
                b.submit_text(lambda feed: None, **kw)
        assert warmed == [] and b.pending.qsize() == 0
        t = b.submit(lambda: None, pitch=-5, gain_db=-6, sample_rate=8000, encoding="flac")
        assert (t.pitch, t.gain_db) == (-5.0, -6.0) and t.flushes
        assert warmed == [(8000, "s16", -5)]   # the pitch's table is designed on the caller's thread
        b.submit(lambda: None, gain_db=-6)
        assert warmed == [(8000, "s16", -5)]   # a gain alone needs no new table
    finally:
        b.close()


def test_window_gets_pitch_and_gain_only_when_not_zero():
    b, calls, warmed = _batcher()
    try:
        for kw, want in ((dict(), {}), (dict(pitch=0.0, gain_db=0.0), {}), (dict(pitch=3), {"pitch": 3.0}),
                         (dict(gain_db=-6, speed=1.5), {"speed": 1.5, "gain_db": -6.0})):
            t = b.submit(lambda: None, **kw)
            calls.clear()
            try:
                b._window(t, None)
            except RuntimeError:
                pass
            assert calls == [want], kw
    finally:
        b.close()


def _server():
    pytest.importorskip("fastapi")
    pytest.importorskip("httpx")
    from fastapi.testclient import TestClient
    spec = importlib.util.spec_from_file_location("openai_server", os.path.join(ROOT, "examples", "openai_server.py"))
    srv = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(srv)
    submitted = []

    class Batcher:
        sched, max_concurrent = [], 0

        def submit(self, prepare, pace=None, speed=1.0, sample_rate=None, encoding="f32", pitch=0.0, gain_db=0.0,
                   **kw):
            submitted.append((speed, pitch, gain_db))
            return iter([(np.zeros(10, dtype=np.int16), sample_rate, {})])

    app = srv.build_app(types.SimpleNamespace(sample_rate=24000), Batcher(), {"v": {"ref_audio": "r.wav"}}, "v")
    return TestClient(app), submitted


def test_server_takes_pitch_and_gain_and_refuses_bad_ones():
    c, submitted = _server()
    for body in ({"pitch": 13}, {"pitch": -12.5}, {"gain_db": 17}, {"gain_db": -100}, {"speed": 0.25, "pitch": 1},
                 {"speed": 4.0, "pitch": -1}, {"pitch": "up"}):
        r = c.post("/v1/audio/speech", json=dict({"input": "hi", "voice": "v"}, **body))
        assert r.status_code in (400, 422), body
    assert submitted == []
    r = c.post("/v1/audio/speech", json={"input": "hi", "voice": "v", "pitch": -2, "gain_db": -6, "speed": 1.25})
    assert r.status_code == 200 and submitted == [(1.25, -2.0, -6.0)]
    c.post("/v1/audio/speech", json={"input": "hi", "voice": "v"})
    assert submitted[-1] == (1.0, 0.0, 0.0)
