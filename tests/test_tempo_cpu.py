"""Speaking-rate control without a GPU: the float64 WSOLA oracle (oracle/tempo_oracle.py) against the host count
function of faster_qwen3_tts/tempo.py, the properties the algorithm promises (exact output length, chunking invariance,
constant in -> constant out, pitch kept), the refusals of out-of-range speeds, and the lead / underrun arithmetic of
ContinuousBatcher at a speaking rate."""
import inspect
import os
import re
import types

import numpy as np
import pytest
import torch

from oracle import prompt_cases  # noqa: F401  (puts the package on sys.path)
from oracle import tempo_oracle as O
from faster_qwen3_tts import tempo as T
from faster_qwen3_tts.model import FasterQwen3TTS
from faster_qwen3_tts.serving import ContinuousBatcher

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPEEDS = (0.25, 0.5, 0.8, 1.25, 2.0, 4.0)
SR = 24000


def test_constants_agree_with_the_c_header():
    h = open(os.path.join(ROOT, "include", "fq3_engine.h")).read()
    val = {k: v for k, v in re.findall(r"#define FQ3_TEMPO_(\w+) ([0-9.e-]+)f?", h)}
    assert int(val["WINDOW"]) == T.WINDOW == O.N and T.HOP == O.H == T.WINDOW // 2
    assert int(val["SEARCH"]) == T.SEARCH == O.D
    assert float(val["EPS"]) == T.EPS == O.EPS
    assert (int(val["Q_MIN"]), int(val["Q_MAX"])) == (T.Q_MIN, T.Q_MAX)


@pytest.mark.parametrize("speed", SPEEDS + (0.3, 3.7))
def test_counts_and_chunking_invariance(speed):
    """the oracle's released samples equal tempo.released for random chunkings (1-sample pushes among them), the
    flushed length is exactly L_out, and the output does not depend on the chunking"""
    rng = np.random.default_rng(int(speed * 100))
    q = T.quantize(speed)
    x = rng.standard_normal(7000) * 0.2
    whole, s = O.stretch(x, speed)
    assert len(whole) == T.out_len(len(x), q) == (len(x) * 1024 + q // 2) // q
    assert len(s.p) == T.frames_run(0, len(x), q, True)
    for mode in ("random", "ones"):
        st, parts, tot, i = O.Wsola(speed), [], 0, 0
        while i < len(x):
            n = 1 if mode == "ones" and i < 1500 else int(rng.integers(1, 900))
            n = min(n, len(x) - i)
            fin = i + n == len(x)
            k0 = len(st.p)
            r = st.push(x[i:i + n], fin)
            assert len(r) == T.released(tot, n, q, fin)
            assert len(st.p) - k0 == T.frames_run(tot, n, q, fin)
            parts.append(r)
            tot, i = tot + n, i + n
        assert np.array_equal(np.concatenate(parts), whole)


def test_c_count_function_agrees(tmp_path):
    """fq3_tempo_released (host code of the extension) against tempo.released, where the library is built"""
    from faster_qwen3_tts.engine import LIB_PATH, load_library
    if not os.path.exists(LIB_PATH):
        pytest.skip("libfq3_engine.so not built")
    lib = load_library()
    rng = np.random.default_rng(1)
    for _ in range(400):
        q = int(rng.integers(T.Q_MIN, T.Q_MAX + 1))
        tot, n, fin = int(rng.integers(0, 50000)), int(rng.integers(0, 20000)), bool(rng.integers(0, 2))
        assert lib.fq3_tempo_released(q, tot, n, int(fin)) == T.released(tot, n, q, fin)
    assert lib.fq3_tempo_released(1024 * 5, 0, 10, 0) == -1


@pytest.mark.parametrize("speed", SPEEDS)
def test_constant_stays_constant(speed):
    """from the first sample on; only the end, where frames reach into the zeros after the input, may differ"""
    y, _ = O.stretch(np.full(6000, 0.3), speed)
    margin = int(np.ceil((O.D + O.N + O.H) / speed)) + O.N
    assert np.abs(y[:len(y) - margin] - 0.3).max() < 1e-12


@pytest.mark.parametrize("speed", (0.5, 0.8, 1.25, 2.0, 4.0))
@pytest.mark.parametrize("f0", (110.0, 220.0, 440.0))
def test_sine_keeps_its_pitch(speed, f0):
    x = 0.5 * np.sin(2 * np.pi * f0 * np.arange(int(2.0 * SR)) / SR)
    y, _ = O.stretch(x, speed)
    core = y[O.N:len(y) - int(np.ceil(2 * O.N / speed)) - O.N]
    spec = np.abs(np.fft.rfft(core * np.hanning(len(core))))
    peak = np.argmax(spec) * SR / len(core)
    assert abs(peak - f0) <= SR / len(core), (peak, f0)


def test_speed_one_is_the_identity():
    x = np.random.default_rng(2).standard_normal(5000)
    y, _ = O.stretch(x, 1.0)
    assert np.array_equal(y, x)
    assert T.released(123, 456, 1024, False) == 456 and T.released(123, 456, 1024, True) == 456
    assert T.tempo_for(1.0) is None and T.tempo_for(1.0 + 1e-6) is None


@pytest.mark.parametrize("speed", (0.2, 0.24, 4.01, 5, 0, -1, float("nan"), float("inf"), "fast", None))
def test_out_of_range_speeds_are_refused(speed):
    with pytest.raises(ValueError, match="speed"):
        T.quantize(speed)


def test_every_generate_method_takes_speed_and_refuses_before_tokenizing():
    class Boom:
        def __getattr__(self, name):
            raise AssertionError(f"touched the model ({name}) before the speed was checked")

    m = FasterQwen3TTS.__new__(FasterQwen3TTS)
    m.model = Boom()
    names = [n for n in dir(FasterQwen3TTS) if n.startswith("generate_")] + ["stream_from_embeds",
                                                                              "stream_batch_from_embeds"]
    assert len(names) == 15
    for name in names:
        p = inspect.signature(getattr(FasterQwen3TTS, name)).parameters
        assert p["speed"].default == 1.0, name
        batch = name == "generate_custom_voice_batch"
        args = [["x"] if batch else "x" for k, v in p.items() if k != "self" and v.default is inspect.Parameter.empty]
        with pytest.raises(ValueError, match="speed"):
            r = getattr(m, name)(*args, speed=9.0)
            if inspect.isgenerator(r):
                next(r)


def test_server_refuses_out_of_range_speed():
    pytest.importorskip("fastapi")
    pytest.importorskip("httpx")
    import importlib.util
    from fastapi.testclient import TestClient
    spec = importlib.util.spec_from_file_location("openai_server", os.path.join(ROOT, "examples", "openai_server.py"))
    srv = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(srv)
    submitted = []

    class Batcher:
        sched, max_concurrent = [], 0

        def submit(self, prepare, pace=None, speed=1.0, **kw):
            submitted.append(speed)
            return iter(())

    model = types.SimpleNamespace(sample_rate=24000)
    app = srv.build_app(model, Batcher(), {"v": {"ref_audio": "r.wav"}}, "v")
    c = TestClient(app)
    for bad in (0.1, 0.249, 4.5):
        r = c.post("/v1/audio/speech", json={"input": "hi", "voice": "v", "speed": bad})
        assert r.status_code == 400 and "speed" in r.text
    assert submitted == []
    r = c.post("/v1/audio/speech", json={"input": "hi", "voice": "v", "speed": 1.5, "response_format": "pcm"})
    assert r.status_code == 200 and submitted == [1.5]


# ---- ContinuousBatcher at a speaking rate, on a fake clock and a fake scheduler ------------------------------------
class _Sched:
    """every request emits `chunk` frames per step until `total`; each step advances the fake clock by `dt`"""

    def __init__(self, clock, dt, total):
        self.clock, self.dt, self.total, self.reqs, self.seen = clock, dt, total, [], []

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
            self.seen.append((rq.tag, rq.due))
            k = min(n, self.total - rq.done)
            rq.done += k
            rq.finished = int(rq.done >= self.total)
            out.append((rq, torch.zeros(k, 16, dtype=torch.long)))
            if rq.finished:
                self.reqs.remove(rq)
        return out


class _Tempo:
    def __init__(self):
        self.closed, self.finals = False, []

    def close(self):
        self.closed = True


class _Win:
    def __init__(self, speed):
        self.tempo = _Tempo() if speed != 1.0 else None

    def push(self, codes, final=False):
        if self.tempo is not None:
            self.tempo.finals.append(final)
        return np.zeros(int(codes.shape[0])), 24000


def _batcher(total, dt):
    clock = [100.0]
    wins, speeds = [], []

    def window(ref_codes, speed=1.0):
        speeds.append(speed)
        wins.append(_Win(speed))
        return wins[-1]
    sched = _Sched(clock, dt, total)
    b = ContinuousBatcher(sched, window, chunk_size=8, frame_s=0.08, lead_high_s=1e9, clock=lambda: clock[0],
                          sleep=lambda s: None)
    return b, sched, wins, speeds, clock


def _prep():
    z = torch.zeros(1, 1, 1)
    return z, z, z, z, None


@pytest.mark.parametrize("speed", (1.0, 0.75, 2.0))
def test_lead_and_underruns_count_audio_at_the_speaking_rate(speed):
    """8 frames (0.64 s of model audio) per 0.5 s step: at speed 1 and 0.75 the listener never runs dry; at speed 2
    a chunk lasts 0.32 s and every chunk after the first finds it dry"""
    b, sched, wins, speeds, clock = _batcher(total=40, dt=0.5)
    try:
        t = b.submit(_prep, pace=1.0, speed=speed)
        chunks = list(t)
    finally:
        b.close()
    assert [c[2]["chunk_steps"] for c in chunks] == [8] * 5
    assert speeds == [speed]
    assert t.underruns == (4 if speed == 2.0 else 0)
    assert t.lead_s == pytest.approx(40 * 0.08 / speed - 1.0 * (clock[0] - t.first_chunk_at))
    assert t.lead_s == 40 * 0.08 / speed - 1.0 * (clock[0] - t.first_chunk_at)
    dues = [d for _, d in sched.seen][1:]
    want = [8 * k * 0.08 / speed - 0.5 * (k - 1) for k in range(1, 5)]
    assert dues == pytest.approx(want)
    if speed == 1.0:
        assert wins[0].tempo is None
    else:
        assert wins[0].tempo.finals == [False] * 4 + [True] and wins[0].tempo.closed


def test_speed_one_lead_is_todays_expression():
    b, sched, wins, speeds, clock = _batcher(total=24, dt=0.3)
    try:
        t = b.submit(_prep, pace=1.25)
        list(t)
    finally:
        b.close()
    assert t.lead_s == t.frames * 0.08 - 1.25 * (clock[0] - t.first_chunk_at)


def test_cancel_drops_the_tempo_state():
    b, sched, wins, speeds, clock = _batcher(total=10 ** 6, dt=0.01)
    try:
        t = b.submit(_prep, pace=None, speed=1.5)
        it = iter(t)
        next(it)
        t.cancel()
        for _ in it:
            pass
    finally:
        b.close()
    assert wins[0].tempo.closed and not len(sched)


def test_submit_refuses_out_of_range_speed():
    b, *_ = _batcher(total=8, dt=0.1)
    try:
        with pytest.raises(ValueError, match="speed"):
            b.submit(_prep, speed=4.5)
        with pytest.raises(ValueError, match="speed"):
            b.submit(_prep, speed=0.1)
    finally:
        b.close()
