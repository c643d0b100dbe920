"""FLAC output without a GPU: the numpy oracle (oracle/flac_oracle.py) against its own RFC 9639 decoder and against
FFmpeg's FLAC decoder, the constants and the buffer bound of faster_qwen3_tts/flac.py and their C twins, the compression
of real Qwen3-TTS speech, and the ``flac`` encoding in the batcher and the example server."""
import ctypes as C
import glob
import importlib.util
import os
import re
import types

import numpy as np
import pytest
import torch

from oracle import prompt_cases  # noqa: F401  (puts the package on sys.path)
from oracle import flac_oracle as O
from faster_qwen3_tts import flac as F
from faster_qwen3_tts.serving import ContinuousBatcher

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _speech():
    return [v.astype(np.int16) for _, v in sorted(np.load(os.path.join(ROOT, "tests", "golden", "speech.npz")).items())]


def _signals():
    rng = np.random.default_rng(11)
    sig = {"speech": _speech()[2][:50000],
           "noise": rng.integers(-32768, 32768, 9000),
           "silence": np.zeros(7000, np.int64),
           "square": np.where(np.arange(9000) % 64 < 32, 32767, -32767)}
    imp = np.zeros(6000, np.int64)
    imp[[0, 1, 777, 4095, 4096, 5999]] = [32767, -32768, 1, -1, 20000, -20000]
    sig["impulses"] = imp
    for n in (1, 15, 16, 17, 255, 256, 257, 4096):
        sig[f"block{n}"] = rng.integers(-32768, 32768, n) >> int(rng.integers(0, 12))
    return {k: np.asarray(v).astype(np.int16) for k, v in sig.items()}


def _chunked(x, rate, sizes):
    st, parts, i = O.Stream(rate), [], 0
    for k, n in enumerate(sizes):
        fin = k == len(sizes) - 1
        bound = F.max_bytes(len(st.carry), n, fin)
        parts.append(st.push(x[i:i + n], fin))
        assert len(parts[-1]) <= bound
        i += n
    return b"".join(parts)


def _random_sizes(rng, total, hi):
    sizes = []
    while sum(sizes) < total:
        sizes.append(min(int(rng.integers(0, hi)), total - sum(sizes)))
    return sizes


def test_constants_agree_with_the_c_header():
    h = open(os.path.join(ROOT, "include", "fq3_engine.h")).read()
    val = {k: int(v) for k, v in re.findall(r"#define FQ3_FLAC_(\w+) (\d+)", h)}
    assert val == {"BLOCK": F.BLOCK, "GRAIN": F.GRAIN, "MAX_ORDER": F.MAX_ORDER,
                   "MAX_PARTITION_ORDER": F.MAX_PARTITION_ORDER, "MAX_K": F.MAX_K, "HEAD_BYTES": F.HEAD_BYTES,
                   "ALIGN": F.ALIGN}
    assert (O.BLOCK, O.GRAIN, O.MAX_ORDER, O.MAX_PARTITION_ORDER, O.MAX_K, O.HEAD_BYTES) == \
        (F.BLOCK, F.GRAIN, F.MAX_ORDER, F.MAX_PARTITION_ORDER, F.MAX_K, F.HEAD_BYTES)
    from faster_qwen3_tts.resample import RATES
    assert O.RATES == RATES and all(r in O.RATE_CODES for r in RATES)
    assert F.ENCODINGS == ("f32", "s16", "ulaw", "alaw", "flac")
    assert len(O.stream_header(24000)) == F.HEAD_BYTES


def test_crc_check_values():
    assert O.crc8(b"123456789") == 0xF4
    assert O.crc16(b"123456789") == 0xFEE8


@pytest.mark.parametrize("rate", (8000, 24000, 44100))
def test_oracle_round_trip(rate):
    """encode -> decode is the identity on every test signal, and the frames follow the blocking rule"""
    for name, x in _signals().items():
        data = O.encode(x, rate)
        y, r, frames = O.decode(data)
        assert r == rate and np.array_equal(y, x), name
        assert [f[1] for f in frames] == [min(O.BLOCK, len(x) - a) for a in range(0, len(x), O.BLOCK)], name
        assert [f[0] for f in frames] == list(range(0, len(x), O.BLOCK)), name
        assert len(data) <= F.max_bytes(0, len(x), True)
        assert int.from_bytes(data[18:26], "big") & ((1 << 36) - 1) == len(x)


def test_subframe_choices():
    """constant and verbatim where they must be, fixed predictors on smooth signals"""
    assert O.choose(np.full(100, -7))[0] == ("constant",)
    rng = np.random.default_rng(1)
    assert O.choose(rng.integers(-32768, 32768, 4096))[0] == ("verbatim",)
    ramp = np.arange(4096) * 3 - 6000
    sub, bits = O.choose(ramp)
    assert sub[0] == "fixed" and sub[1] == 2 and bits < 8 + 16 * 4096 // 10   # second difference is zero
    for n, o in ((17, 0), (16, 4)):
        assert O.partition_orders(n, o) == ([0] if n == 17 else [0, 1])   # 16 >> 2 = 4 is not more than 4


@pytest.mark.parametrize("rate", (16000, 24000, 48000))
def test_decoded_samples_do_not_depend_on_the_chunking(rate):
    rng = np.random.default_rng(rate)
    x = np.concatenate([_speech()[0][:40000], rng.integers(-32768, 32768, 2000).astype(np.int16), np.zeros(3000, np.int16)])
    whole = O.encode(x, rate)
    for hi in (9000, 700, 40):
        sizes = _random_sizes(rng, len(x), hi)
        data = _chunked(x, rate, sizes)
        y, r, frames = O.decode(data)
        assert np.array_equal(y, x) and r == rate
        assert int.from_bytes(data[18:26], "big") & ((1 << 36) - 1) == (len(x) if len(sizes) == 1 else 0)
        assert all(n % O.GRAIN == 0 for _, n, _, _ in frames[:-1])
        if len(sizes) > 1:
            assert data != whole   # the bytes follow the pushes; the samples do not


def test_compression_of_speech():
    """on real Qwen3-TTS speech at 24 kHz the stream is at most 0.52 of the s16 bytes"""
    files = _speech()
    total = sum(len(O.encode(x, 24000)) for x in files)
    s16 = sum(2 * len(x) for x in files)
    print(f"FLAC / s16 on the speech fixture: {total / s16:.4f}")
    assert total <= 0.52 * s16


def _lib():
    from faster_qwen3_tts.engine import LIB_PATH, load_library
    if not os.path.exists(LIB_PATH):
        pytest.skip("the extension is not built")
    return load_library()


def test_max_bytes_c_python_and_oracle_agree():
    lib = _lib()
    rng = np.random.default_rng(0)
    for _ in range(3000):
        c, n, f = int(rng.integers(0, 16)), int(rng.integers(0, 10 ** 6)), bool(rng.integers(0, 2))
        assert lib.fq3_flac_max_bytes(c, n, int(f)) == F.max_bytes(c, n, f) == O.max_bytes(c, n, f)
    for c in range(16):
        for n in range(40):
            for f in (0, 1):
                assert lib.fq3_flac_max_bytes(c, n, f) == F.max_bytes(c, n, bool(f))
    assert lib.fq3_flac_max_bytes(16, 1, 0) == lib.fq3_flac_max_bytes(-1, 1, 0) == lib.fq3_flac_max_bytes(0, -1, 0) == -1


# ---- an independent decoder: FFmpeg's, from the libraries opencv-python-headless bundles ------------------------------
def _ffmpeg():
    try:
        import cv2
    except ImportError:
        pytest.skip("FFmpeg's FLAC decoder not found: opencv-python-headless (which bundles libavcodec) is not installed")
    d = os.path.join(os.path.dirname(os.path.dirname(cv2.__file__)), "opencv_python_headless.libs")
    found = glob.glob(os.path.join(d, "libavcodec-*"))
    if not found:
        pytest.skip(f"FFmpeg's FLAC decoder not found: no libavcodec in {d}")
    try:
        for pre in ("libcrypto", "libssl", "libdrm", "libavutil", "libswresample", "libvpx", "libaom"):
            for f in glob.glob(os.path.join(d, pre + "-*")):
                C.CDLL(f, mode=C.RTLD_GLOBAL)
        av = C.CDLL(found[0])
    except OSError as ex:
        pytest.skip(f"FFmpeg's FLAC decoder not found: libavcodec does not load ({ex})")
    for f in ("avcodec_find_decoder_by_name", "avcodec_alloc_context3", "av_packet_alloc", "av_frame_alloc"):
        getattr(av, f).restype = C.c_void_p
    av.avcodec_alloc_context3.argtypes = [C.c_void_p]
    av.avcodec_open2.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    av.av_new_packet.argtypes = [C.c_void_p, C.c_int]
    av.avcodec_send_packet.argtypes = [C.c_void_p, C.c_void_p]
    av.avcodec_receive_frame.argtypes = [C.c_void_p, C.c_void_p]
    for f in ("av_packet_unref", "av_frame_unref", "avcodec_free_context", "av_packet_free", "av_frame_free"):
        getattr(av, f).argtypes = [C.c_void_p]
    if not av.avcodec_find_decoder_by_name(b"flac"):
        pytest.skip("FFmpeg's FLAC decoder not found: this libavcodec has no flac decoder")
    return av


def _ffmpeg_decode(av, data):
    """the stream header as the first packet, then one packet per frame; AVFrame's data[0] / nb_samples / format are at
    offsets 0 / 112 / 116, AVPacket's data at 24 (layouts stable since FFmpeg 4)"""
    codec = av.avcodec_find_decoder_by_name(b"flac")
    ctx = C.c_void_p(av.avcodec_alloc_context3(codec))
    assert av.avcodec_open2(ctx, codec, None) == 0
    pkt, frm = C.c_void_p(av.av_packet_alloc()), C.c_void_p(av.av_frame_alloc())
    _, _, frames = O.decode(data)
    pieces = [data[:frames[0][2] if frames else len(data)]] + [data[p:p + n] for _, _, p, n in frames]
    out = []

    def drain():
        while av.avcodec_receive_frame(ctx, frm) == 0:
            ns = C.c_int.from_address(frm.value + 112).value
            assert C.c_int.from_address(frm.value + 116).value in (1, 6)   # AV_SAMPLE_FMT_S16 / S16P
            ptr = C.c_void_p.from_address(frm.value).value
            out.append(np.frombuffer((C.c_int16 * ns).from_address(ptr), np.int16).copy())
            av.av_frame_unref(frm)
    try:
        for piece in pieces:
            assert av.av_new_packet(pkt, len(piece)) == 0
            C.memmove(C.c_void_p.from_address(pkt.value + 24).value, piece, len(piece))
            assert av.avcodec_send_packet(ctx, pkt) == 0
            av.av_packet_unref(pkt)
            drain()
        av.avcodec_send_packet(ctx, None)
        drain()
    finally:
        av.av_frame_free(C.byref(frm))
        av.av_packet_free(C.byref(pkt))
        av.avcodec_free_context(C.byref(ctx))
    return np.concatenate(out) if out else np.zeros(0, np.int16)


def test_ffmpeg_decodes_the_same_samples():
    av = _ffmpeg()
    rng = np.random.default_rng(5)
    for rate in (8000, 22050, 48000):
        for name, x in _signals().items():
            assert np.array_equal(_ffmpeg_decode(av, O.encode(x, rate)), x), (rate, name)
        x = _speech()[1][:30000]
        data = _chunked(x, rate, _random_sizes(rng, len(x), 3000))
        assert np.array_equal(_ffmpeg_decode(av, data), x), rate


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
    """8 frames of 1920 samples at 24 kHz -> that many at the window's rate as s16, or the oracle's FLAC of them"""

    def __init__(self, sample_rate=None, encoding="f32"):
        self.rate, self.encoding = sample_rate or 24000, encoding
        self.resampler = _Stage()
        self.flac = _Stage() if encoding == "flac" else None
        self.stream = O.Stream(self.rate) if encoding == "flac" else None

    def push(self, codes, final=False):
        self.resampler.finals.append(final)
        x = (np.arange(int(codes.shape[0]) * 1920 * self.rate // 24000) % 200 - 100).astype(np.int16)
        if self.flac is None:
            return x, self.rate
        self.flac.finals.append(final)
        return np.frombuffer(self.stream.push(x, final), np.uint8), self.rate


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


@pytest.mark.parametrize("rate", (None, 8000, 44100))
def test_flac_tickets_are_accepted_and_keep_the_s16_lead(rate):
    """a flac ticket's window gets the encoding, its FLAC stage flushes with the last chunk and returns to its pool,
    the ticket's audio is one complete stream, and the listener's lead is that of the same ticket in s16"""
    leads = {}
    for enc in ("s16", "flac"):
        b, wins, calls, clock = _batcher(total=40, dt=0.5)
        try:
            t = b.submit(_prep, pace=1.0, sample_rate=rate, encoding=enc)
            chunks = list(t)
            end = clock[0]
        finally:
            b.close()
        leads[enc] = (t.lead_s, t.underruns, [c[2]["chunk_steps"] for c in chunks], end - t.first_chunk_at)
        assert calls == [{"sample_rate": rate or 24000, "encoding": enc}]
        assert all(c[1] == (rate or 24000) for c in chunks)
        if enc == "flac":
            assert wins[0].flac.finals == [False] * 4 + [True] and wins[0].flac.closed
            data = np.concatenate([c[0] for c in chunks])
            assert data.dtype == np.uint8
            y, r, _ = O.decode(data.tobytes())
            assert r == (rate or 24000) and len(y) == 40 * 1920 * (rate or 24000) // 24000
    assert leads["flac"] == leads["s16"]


def test_submit_refuses_unknown_encodings():
    b, *_ = _batcher(total=8, dt=0.1)
    try:
        for bad in ("mp3", "opus", "FLAC", None):
            with pytest.raises(ValueError, match="encoding"):
                b.submit(_prep, encoding=bad)
        with pytest.raises(ValueError, match="sample_rate"):
            b.submit(_prep, sample_rate=11025, encoding="flac")
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
    x = (np.arange(5000) % 300 - 150).astype(np.int16)

    class Batcher:
        """hands back the oracle's FLAC of a fixed s16 signal in two chunks"""
        sched, max_concurrent = [], 0

        def submit(self, prepare, pace=None, speed=1.0, sample_rate=None, encoding="f32", **kw):
            submitted.append((sample_rate, encoding))
            st = O.Stream(sample_rate)
            return iter([(np.frombuffer(st.push(x[:3000]), np.uint8), sample_rate, {}),
                         (np.frombuffer(st.push(x[3000:], True), np.uint8), sample_rate, {})])

    app = srv.build_app(types.SimpleNamespace(sample_rate=24000), Batcher(), {"v": {"ref_audio": "r.wav"}}, "v")
    return TestClient(app), submitted, x


@pytest.mark.parametrize("rate", (24000, 8000, 48000))
def test_server_serves_flac(rate):
    c, submitted, x = _server()
    body = {"input": "hi", "voice": "v", "response_format": "flac"}
    if rate != 24000:
        body["sample_rate"] = rate
    r = c.post("/v1/audio/speech", json=body)
    assert r.status_code == 200 and r.headers["content-type"] == "audio/flac"
    assert submitted == [(rate, "flac")]
    y, sr, _ = O.decode(r.content)
    assert sr == rate and np.array_equal(y, x)


def test_server_still_refuses_unknown_formats():
    c, submitted, _ = _server()
    for fmt in ("mp3", "opus", "aac", "f32"):
        r = c.post("/v1/audio/speech", json={"input": "hi", "voice": "v", "response_format": fmt})
        assert r.status_code == 400 and "flac" in r.json()["detail"], fmt
    assert submitted == []
