"""Output rate and encoding without a GPU: the float64 oracle (oracle/resample_oracle.py) against scipy's filter design
and polyphase resampler and against the standard library's G.711, the host count function of
faster_qwen3_tts/resample.py and its C twin, chunking invariance, the refusals of unknown rates and encodings by every
generate method, the batcher and the example server, and the listener's lead at every rate."""
import ctypes as C
import importlib.util
import inspect
import os
import re
import types
import warnings

import numpy as np
import pytest
import torch

from oracle import prompt_cases  # noqa: F401  (puts the package on sys.path)
from oracle import resample_oracle as O
from faster_qwen3_tts import resample as R
from faster_qwen3_tts.model import FasterQwen3TTS
from faster_qwen3_tts.serving import ContinuousBatcher, to_pcm16

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RATIOS = {8000: (1, 3), 16000: (2, 3), 22050: (147, 160), 24000: (1, 1), 32000: (4, 3), 44100: (147, 80),
          48000: (2, 1)}
TAPS_PER_OUTPUT = {8000: 193, 16000: 97, 22050: 70, 32000: 65, 44100: 65, 48000: 65}
BAD_RATES = (0, -8000, 11025, 96000, 8000.5, "8000", None.__class__, True)


def _audioop():
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        return pytest.importorskip("audioop")


def test_constants_agree_with_the_c_header():
    h = open(os.path.join(ROOT, "include", "fq3_engine.h")).read()
    val = dict(re.findall(r"#define FQ3_RESAMPLE_(\w+) ([0-9.]+)", h))
    assert int(val["IN_RATE"]) == R.IN_RATE == O.IN_RATE
    assert int(val["HALF_PER_M"]) == R.HALF_PER_M == O.HALF_PER_M
    assert float(val["CUTOFF"]) == R.CUTOFF == O.CUTOFF and float(val["BETA"]) == R.BETA == O.BETA
    assert int(val["ALIGN"]) == R.ALIGN
    enc = {k.lower(): int(v) for k, v in re.findall(r"#define FQ3_ENC_(\w+) (\d+)", h)}
    assert enc == R.ENCODINGS
    assert R.RATES == O.RATES == tuple(RATIOS)


@pytest.mark.parametrize("rate", R.RATES)
def test_ratios_and_taps(rate):
    L, M, half = R.ratio(rate)
    assert (L, M) == RATIOS[rate] and (L, M, half) == O.ratio(rate)
    if rate != 24000:
        assert half == 32 * max(L, M)
        assert max(len(O.reads(n, rate)) for n in range(1000, 1000 + L)) == TAPS_PER_OUTPUT[rate]
    assert 2 * half + 1 <= 10241


@pytest.mark.parametrize("rate", R.RATES)
def test_oracle_design_is_firwin_and_output_is_resample_poly(rate):
    signal = pytest.importorskip("scipy.signal")
    L, M, half = O.ratio(rate)
    h = O.design(rate)
    if half:
        want = signal.firwin(2 * half + 1, 0.9 / max(L, M), window=("kaiser", 8.6))
        assert np.abs(h - want).max() <= 1e-15
        assert abs(h.sum() - 1) < 1e-12
    else:
        assert np.array_equal(h, [1.0])
    rng = np.random.default_rng(rate)
    for n in (1, 37, 2400):
        x = rng.standard_normal(n)
        y = O.resample(x, rate)
        ref = signal.resample_poly(x, L, M, window=h)
        assert len(y) == len(ref) == -(-n * L // M)
        assert np.abs(y - ref).max() <= 1e-12


@pytest.mark.parametrize("rate", R.RATES)
def test_counts_and_chunking_invariance(rate):
    """the oracle's streaming releases exactly resample.released per push (random splits, 1-sample pushes), reads only
    input that exists, and its output does not depend on the chunking"""
    rng = np.random.default_rng(rate + 1)
    x = rng.standard_normal(1500)
    whole = O.resample(x, rate)
    for mode in ("random", "ones"):
        st, parts, tot, i = O.Stream(rate), [], 0, 0
        while i < len(x):
            n = 1 if mode == "ones" and i < 400 else int(rng.integers(0, 300))
            n = min(n, len(x) - i)
            fin = i + n == len(x)
            r = st.push(x[i:i + n], fin)
            assert len(r) == R.released(tot, n, rate, fin)
            parts.append(r)
            tot, i = tot + n, i + n
        assert np.array_equal(np.concatenate(parts), whole)
    # released outputs read only pushed input; the look-ahead is half / L input samples
    L, M, half = R.ratio(rate)
    for T in (0, 1, 5, 97, 500, 12345):
        e = R.emitted(T, rate, False)
        assert (e == 0 or O.reads(e - 1, rate)[0] < T) and O.reads(e, rate)[0] >= T
    assert half / L / 24000 <= {8000: 0.004, 16000: 0.002}.get(rate, 0.0015)


def _lib():
    from faster_qwen3_tts.engine import LIB_PATH, load_library
    if not os.path.exists(LIB_PATH):
        pytest.skip("the extension is not built")
    return load_library()


@pytest.mark.parametrize("rate", R.RATES)
def test_c_design_and_counts_agree(rate):
    """fq3_resample_taps / fq3_resample_released (host code of the extension) against the oracle and resample.py"""
    lib = _lib()
    n = lib.fq3_resample_taps(rate, None, 0)
    buf = (C.c_double * n)()
    assert lib.fq3_resample_taps(rate, buf, n) == n == 2 * R.ratio(rate)[2] + 1
    assert np.abs(np.frombuffer(buf, dtype=np.float64) - O.design(rate)).max() <= 1e-14
    rng = np.random.default_rng(rate)
    for _ in range(3000):
        t, m, f = int(rng.integers(0, 10 ** 6)), int(rng.integers(0, 20000)), bool(rng.integers(0, 2))
        assert lib.fq3_resample_released(rate, t, m, int(f)) == R.released(t, m, rate, f)
    for t in range(200):
        for m in range(4):
            assert lib.fq3_resample_released(rate, t, m, 0) == R.released(t, m, rate, False)
    assert lib.fq3_resample_released(11025, 0, 1, 0) == -1 and lib.fq3_resample_taps(11025, None, 0) == -1


def test_g711_matches_audioop_on_every_s16_value():
    audioop = _audioop()
    s = np.arange(-32768, 32768, dtype=np.int16)
    assert np.array_equal(O.lin2ulaw(s), np.frombuffer(audioop.lin2ulaw(s.tobytes(), 2), np.uint8))
    assert np.array_equal(O.lin2alaw(s), np.frombuffer(audioop.lin2alaw(s.tobytes(), 2), np.uint8))


def test_s16_rule_is_to_pcm16():
    rng = np.random.default_rng(3)
    y = np.concatenate([rng.standard_normal(5000) * 0.5, [-1.5, -1.0, -0.99999, 0.0, 0.99999, 1.0, 1.5],
                        np.arange(-40000, 40000, 7) / 32768.0]).astype(np.float32)
    assert O.to_s16(y).tobytes() == to_pcm16(y)


@pytest.mark.parametrize("rate", BAD_RATES)
def test_unknown_rates_are_refused(rate):
    with pytest.raises(ValueError, match="sample_rate"):
        R.check_rate(rate)


def test_identity_and_known_rates():
    assert R.check_rate(None) == 24000 and R.check_rate(8000.0) == 8000 and R.check_rate(np.int64(44100)) == 44100
    assert R.resampler_for(None) is None and R.resampler_for(24000, "f32") is None
    for bad in ("mp3", "pcm", None):
        with pytest.raises(ValueError, match="encoding"):
            R.check_encoding(bad)
    for T in (0, 1, 1000):
        assert R.emitted(T, 24000, False) == R.emitted(T, 24000, True) == T


def test_every_generate_method_takes_sample_rate_and_refuses_before_tokenizing():
    class Boom:
        def __getattr__(self, name):
            raise AssertionError(f"touched the model ({name}) before the sample rate was checked")

    m = FasterQwen3TTS.__new__(FasterQwen3TTS)
    m.model = Boom()
    names = [n for n in dir(FasterQwen3TTS) if n.startswith("generate_")] + ["stream_from_embeds",
                                                                              "stream_batch_from_embeds"]
    assert len(names) == 15
    for name in names:
        p = inspect.signature(getattr(FasterQwen3TTS, name)).parameters
        assert p["sample_rate"].default is None, name
        batch = name == "generate_custom_voice_batch"
        args = [["x"] if batch else "x" for k, v in p.items() if k != "self" and v.default is inspect.Parameter.empty]
        for bad in (11025, 96000):
            with pytest.raises(ValueError, match="sample_rate"):
                r = getattr(m, name)(*args, sample_rate=bad)
                if inspect.isgenerator(r):
                    next(r)


def test_text_streaming_takes_sample_rate():
    from faster_qwen3_tts.text_stream import generate_text_streaming
    assert inspect.signature(generate_text_streaming).parameters["sample_rate"].default is None


# ---- ContinuousBatcher and the server, on fakes -------------------------------------------------------------------
class _Sched:
    def __init__(self, clock, dt, total):
        self.clock, self.dt, self.total, self.reqs = clock, dt, total, []

    def has_capacity(self):
        return True

    def submit(self, tie, tam, tth, tpe, tag, **kw):
        rq = types.SimpleNamespace(tag=tag, finished=0, done=0, due=0.0, hold=False)
        self.reqs.append(rq)
        return rq

    def cancel(self, rq):
        self.reqs.remove(rq)

    def __len__(self):
        return len(self.reqs)

    def step(self, n):
        self.clock[0] += self.dt
        out = []
        for rq in list(self.reqs):
            k = min(n, self.total - rq.done)
            rq.done += k
            rq.finished = int(rq.done >= self.total)
            out.append((rq, torch.zeros(k, 16, dtype=torch.long)))
            if rq.finished:
                self.reqs.remove(rq)
        return out


class _Stage:
    def __init__(self):
        self.closed, self.finals = False, []

    def close(self):
        self.closed = True


class _Win:
    """8 frames of 1920 samples at 24 kHz -> that many at the window's rate, in its encoding"""

    def __init__(self, sample_rate=None, encoding="f32"):
        self.rate = sample_rate or 24000
        self.dtype = {"f32": np.float32, "s16": np.int16}.get(encoding, np.uint8)
        self.resampler = _Stage() if sample_rate is not None else None

    def push(self, codes, final=False):
        if self.resampler is not None:
            self.resampler.finals.append(final)
        return np.zeros(int(codes.shape[0]) * 1920 * self.rate // 24000, dtype=self.dtype), self.rate


def _batcher(total, dt):
    clock, wins, calls = [100.0], [], []

    def window(ref_codes, **kw):
        calls.append(kw)
        wins.append(_Win(**kw))
        return wins[-1]
    b = ContinuousBatcher(_Sched(clock, dt, total), window, chunk_size=8, frame_s=0.08, lead_high_s=1e9,
                          clock=lambda: clock[0], sleep=lambda s: None)
    return b, wins, calls, clock


def _prep():
    z = torch.zeros(1, 1, 1)
    return z, z, z, z, None


@pytest.mark.parametrize("rate,encoding", [(None, "f32"), (8000, "ulaw"), (16000, "s16"), (48000, "f32"),
                                           (24000, "s16"), (44100, "alaw")])
def test_lead_is_the_same_at_every_rate(rate, encoding):
    """8 frames (0.64 s) per 0.5 s step: the lead counts audio seconds, whatever the rate and the encoding"""
    b, wins, calls, clock = _batcher(total=40, dt=0.5)
    try:
        t = b.submit(_prep, pace=1.0, sample_rate=rate, encoding=encoding)
        chunks = list(t)
        end = clock[0]
        a = b.submit(_prep, sample_rate=rate, encoding=encoding).audio()
    finally:
        b.close()
    assert [c[2]["chunk_steps"] for c in chunks] == [8] * 5 and t.underruns == 0
    assert t.lead_s == 40 * 0.08 - 1.0 * (end - t.first_chunk_at)
    identity = (rate or 24000, encoding) == (24000, "f32")
    assert calls == [{} if identity else {"sample_rate": rate, "encoding": encoding}] * 2
    assert all(c[1] == (rate or 24000) for c in chunks)
    assert a.dtype == wins[0].dtype and len(a) == 40 * 1920 * (rate or 24000) // 24000
    if not identity:
        assert wins[0].resampler.finals == [False] * 4 + [True] and wins[0].resampler.closed


def test_submit_refuses_unknown_rates_and_encodings():
    b, *_ = _batcher(total=8, dt=0.1)
    try:
        with pytest.raises(ValueError, match="sample_rate"):
            b.submit(_prep, sample_rate=11025)
        with pytest.raises(ValueError, match="encoding"):
            b.submit(_prep, encoding="mp3")
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
        """hands back one chunk of the request's encoding, made from a fixed float32 signal the way the device does"""
        sched, max_concurrent = [], 0

        def submit(self, prepare, pace=None, speed=1.0, sample_rate=None, encoding="f32", **kw):
            submitted.append((sample_rate, encoding))
            y = np.linspace(-1.2, 1.2, 999, dtype=np.float32)
            return iter([(O.encode(y, encoding), sample_rate, {})])

    app = srv.build_app(types.SimpleNamespace(sample_rate=24000), Batcher(), {"v": {"ref_audio": "r.wav"}}, "v")
    return TestClient(app), submitted


def test_server_refuses_unknown_rates_and_formats():
    c, submitted = _server()
    for body in ({"sample_rate": 11025}, {"sample_rate": 96000}, {"response_format": "mp3"},
                 {"response_format": "f32"}):
        r = c.post("/v1/audio/speech", json=dict({"input": "hi", "voice": "v"}, **body))
        assert r.status_code == 400, body
    assert submitted == []


@pytest.mark.parametrize("fmt,rate", [("wav", 24000), ("wav", 8000), ("pcm", 24000), ("pcm", 48000), ("ulaw", 8000),
                                      ("alaw", 16000)])
def test_server_asks_the_batcher_for_the_response_encoding(fmt, rate):
    """the default wav / pcm at 24 kHz is s16 on the device and equals today's to_pcm16 bytes; the header carries the
    requested rate; ulaw / alaw are raw G.711 bytes"""
    c, submitted = _server()
    body = {"input": "hi", "voice": "v", "response_format": fmt}
    if rate != 24000:
        body["sample_rate"] = rate
    r = c.post("/v1/audio/speech", json=body)
    assert r.status_code == 200
    enc = {"wav": "s16", "pcm": "s16"}.get(fmt, fmt)
    assert submitted == [(rate, enc)]
    y = np.linspace(-1.2, 1.2, 999, dtype=np.float32)
    data = r.content
    if fmt == "wav":
        assert data[:4] == b"RIFF" and int.from_bytes(data[24:28], "little") == rate
        assert int.from_bytes(data[28:32], "little") == 2 * rate
        data = data[44:]
    if enc == "s16":
        assert data == to_pcm16(y)
    else:
        audioop = _audioop()
        want = (audioop.lin2ulaw if fmt == "ulaw" else audioop.lin2alaw)(to_pcm16(y), 2)
        assert data == want


@pytest.mark.parametrize("speed", (1.0004, 0.9996, 1.0))
def test_one_shot_and_takes_at_a_speed_that_quantises_to_one(speed):
    """a speed within 1/2048 of 1 passes the speed check and is the identity: the one-shot and takes deliveries return
    the codec's 24 kHz audio unchanged, with no tempo created (no device needed)"""
    from faster_qwen3_tts import tempo as T
    assert T.quantize(speed) == T.Q_ONE

    class Codec:
        def decode(self, inputs):
            codes = inputs["audio_codes"]
            return [torch.arange(c.shape[0] * 1920, dtype=torch.float32) / 1e5 for c in codes], 24000

    m = FasterQwen3TTS.__new__(FasterQwen3TTS)
    m.sample_rate = 24000
    codes = [torch.zeros(5, 16, dtype=torch.long), None, torch.zeros(7, 16, dtype=torch.long)]
    want, _ = m._decode_takes(Codec(), codes, None)
    got, sr = m._decode_takes(Codec(), codes, None, speed=speed)
    assert sr == 24000 and all(np.array_equal(g, w) for g, w in zip(got, want))
    (one,), sr = m._decode_all(Codec(), codes[0], None, speed=speed)
    assert sr == 24000 and np.array_equal(one, want[0])
