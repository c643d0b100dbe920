"""GPU tests of the FLAC stage (csrc/fq3_flac.cu through faster_qwen3_tts/flac.py).

The kernel's bytes equal the numpy oracle's (oracle/flac_oracle.py) bit for bit: for every test signal and rate, for
random push sequences, and for streams sharing a launch against each alone.  Bad input is refused before any launch.
End to end on the synthetic model: a ``flac`` ticket's bytes decode to exactly the samples of an ``s16`` ticket of the
same request (both codec policies, 8 and 24 kHz, speeds 1 and 1.5, tickets of both encodings in the same steps), and
``flac.convert`` of a one-shot output decodes to that output's s16."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import prompt_cases  # noqa: F401  (puts the package on sys.path)
from oracle import flac_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RATES = (8000, 16000, 22050, 24000, 32000, 44100, 48000)


def _speech():
    return [v.astype(np.int16) for _, v in sorted(np.load(os.path.join(ROOT, "tests", "golden", "speech.npz")).items())]


def _signals():
    rng = np.random.default_rng(7)
    sig = {"speech": _speech()[0][20000:60000],
           "noise": rng.integers(-32768, 32768, 9000),
           "silence": np.zeros(5000, np.int64),
           "square": np.where(np.arange(9000) % 96 < 48, 32767, -32767)}
    imp = np.zeros(6000, np.int64)
    imp[[0, 1, 777, 4095, 4096, 5999]] = [32767, -32768, 1, -1, 20000, -20000]
    sig["impulses"] = imp
    for n in (1, 15, 16, 17, 255, 256, 257, 4096):
        sig[f"block{n}"] = rng.integers(-300, 300, n)
    return {k: np.asarray(v).astype(np.int16) for k, v in sig.items()}


def _dev(x):
    return torch.as_tensor(np.asarray(x, dtype=np.int16), device="cuda")


def _bytes(t):
    return t.cpu().numpy().tobytes()


def _pushes(x, rate, sizes):
    """the GPU's bytes and the oracle's bytes of x pushed in the given sizes, flushed with the last"""
    from faster_qwen3_tts import flac as F
    e, st = F.Encoder(rate, "cuda"), O.Stream(rate)
    got, want, i = [], [], 0
    for k, n in enumerate(sizes):
        fin = k == len(sizes) - 1
        bound = F.max_bytes(e.carried, n, fin)
        out = F.process([e], [_dev(x[i:i + n])], fin)[0]
        assert out.numel() <= bound
        got.append(_bytes(out))
        want.append(st.push(x[i:i + n], fin))
        i += n
    e.close()
    return got, want


@pytest.mark.parametrize("rate", RATES)
def test_kernel_bytes_equal_the_oracle(rate):
    from faster_qwen3_tts import flac as F
    for name, x in _signals().items():
        got = _bytes(F.convert(_dev(x), rate))
        assert got == O.encode(x, rate), (rate, name)
        y, r, _ = O.decode(got)
        assert r == rate and np.array_equal(y, x), (rate, name)


@pytest.mark.parametrize("rate", (8000, 24000, 44100))
def test_random_push_sequences(rate):
    rng = np.random.default_rng(rate)
    x = np.concatenate([_speech()[1][:30000], rng.integers(-32768, 32768, 3000).astype(np.int16)])
    for trial in range(4):
        sizes = []
        while sum(sizes) < len(x):
            sizes.append(min(int(rng.integers(0, 9000 if trial < 2 else 40)), len(x) - sum(sizes)))
            if trial >= 2 and len(sizes) > 200:
                sizes.append(len(x) - sum(sizes))
        got, want = _pushes(x, rate, sizes)
        assert got == want, (rate, trial)
        assert np.array_equal(O.decode(b"".join(got))[0], x)


def test_streams_in_one_launch_equal_each_alone():
    from faster_qwen3_tts import flac as F
    rng = np.random.default_rng(0)
    speech = np.concatenate(_speech())
    rates = [8000, 48000, 22050, 24000, 44100, 16000, 32000, 24000]
    sigs = [speech[i * 37000:i * 37000 + 20000 + 3111 * i] for i in range(len(rates))]
    sigs[3] = np.zeros(9000, np.int16)
    encs = [F.Encoder(r, "cuda") for r in rates]
    parts = [[] for _ in rates]
    pushed = [[] for _ in rates]
    pos = [0] * len(rates)
    while any(p < len(x) for p, x in zip(pos, sigs)):   # own push lengths (empty ones among them) and flush points
        live = [i for i in range(len(rates)) if pos[i] < len(sigs[i])]
        ns = [min(int(rng.integers(0, 12000)), len(sigs[i]) - pos[i]) for i in live]
        outs = F.process([encs[i] for i in live], [_dev(sigs[i][pos[i]:pos[i] + n]) for i, n in zip(live, ns)],
                         [pos[i] + n == len(sigs[i]) for i, n in zip(live, ns)])
        for i, n, o in zip(live, ns, outs):
            parts[i].append(_bytes(o))
            pushed[i].append(n)
            pos[i] += n
    for i, e in enumerate(encs):
        e.close()
        alone, want = _pushes(sigs[i], rates[i], pushed[i])
        assert parts[i] == alone == want, rates[i]


def test_bad_input_is_refused_before_any_launch():
    from faster_qwen3_tts import flac as F
    from faster_qwen3_tts.engine import load_library
    lib = load_library()
    h = C.c_void_p()
    for rate in (11025, 96000, 0):
        assert lib.fq3_flac_create(0, rate, C.byref(h)) == -1
    a, b = F.Encoder(8000, "cuda"), F.Encoder(48000, "cuda")
    x = _dev(np.arange(2000) - 1000)
    out = torch.empty(16384, dtype=torch.uint8, device="cuda")
    lens_dev = torch.zeros(2, dtype=torch.int32, device="cuda")
    lens, fl = (C.c_int64 * 2)(1000, 1000), (C.c_int32 * 2)(0, 0)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(handles, inp, outp, cap=16384, ol=None):
        arr = (C.c_void_p * len(handles))(*[t._h for t in handles])
        return lib.fq3_flac_process(arr, len(handles), inp, lens, fl, outp, cap,
                                    C.c_void_p(lens_dev.data_ptr()) if ol is None else ol, stream)

    xp, op = C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr())
    assert call([a, a], xp, op) == -1 and b"twice" in lib.fq3_flac_last_error()
    assert call([a, b], None, op) == -1
    assert call([a, b], C.c_void_p(x.data_ptr() + 1), op) == -1 and b"misaligned" in lib.fq3_flac_last_error()
    assert call([a, b], xp, C.c_void_p(out.data_ptr() + 4)) == -1 and b"misaligned" in lib.fq3_flac_last_error()
    assert call([a, b], xp, op, ol=C.c_void_p(lens_dev.data_ptr() + 2)) == -1
    assert call([a, b], xp, op, ol=C.c_void_p(None)) == -1
    assert call([a, b], xp, op, cap=2000) == -1 and b"smaller" in lib.fq3_flac_last_error()
    assert call([a, b], xp, None) == -1
    torch.cuda.synchronize()
    assert lens_dev.tolist() == [0, 0]   # nothing was launched
    y = np.arange(3000) % 50 - 25
    assert _bytes(F.process([a], [_dev(y)], True)[0]) == O.encode(y, 8000)   # state untouched
    a = F.Encoder(8000, "cuda")
    with pytest.raises(ValueError, match="twice"):
        F.process([a, a], [x, x], False)
    with pytest.raises(ValueError, match="int16"):
        F.process([a], [x.float()], False)
    F.process([a], [x], True)
    with pytest.raises(ValueError, match="flushed"):
        F.process([a], [x], False)
    assert lib.fq3_flac_process((C.c_void_p * 1)(a._h), 1, xp, lens, (C.c_int32 * 1)(0), op, 16384,
                                C.c_void_p(lens_dev.data_ptr()), stream) == -3
    a.close()
    b.close()
    c = F.Encoder(8000, "cuda")   # a flushed handle from the pool starts a new stream
    assert _bytes(F.process([c], [_dev(y)], True)[0]) == O.encode(y, 8000)
    c.close()


# ---- end to end on the synthetic model --------------------------------------------------------------------------------
def _model(max_batch=8):
    from faster_qwen3_tts import FasterQwen3TTS
    m = FasterQwen3TTS.from_synthetic("tiny", dtype=torch.bfloat16, max_seq_len=512, seed=5, max_batch=max_batch)
    m.predictor_graph.do_sample = False
    return m


GEN = dict(max_new_tokens=21, min_new_tokens=21, do_sample=False)


@pytest.mark.parametrize("codec_mode", ["window", "stateful"])
def test_flac_tickets_decode_to_the_s16_tickets(codec_mode, monkeypatch):
    """pairs of the same request, one flac and one s16, submitted together so that both encodings share steps"""
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    import time
    from faster_qwen3_tts.serving import batcher_for_model, voice_clone_request
    m = _model()
    m.streaming_codec = codec_mode
    texts = ["hello there general kenobi", "short one", "the quick brown fox jumps", "another request here"]
    outs = [(8000, 1.0), (8000, 1.5), (24000, 1.0), (None, 1.5)]
    b = batcher_for_model(m, chunk_size=8)
    try:
        tickets = []
        for i, (text, (rate, speed)) in enumerate(zip(texts, outs)):
            for enc in ("flac", "s16"):
                tickets.append(b.submit(voice_clone_request(m, text, "English", "ref.wav", "ref words",
                                                            xvec_only=(i % 2 == 0)),
                                        sample_rate=rate, encoding=enc, speed=speed, **GEN))
            time.sleep(0.05)   # staggered arrivals
        audio = [t.audio() for t in tickets]
    finally:
        b.close()
    for i, (rate, speed) in enumerate(outs):
        flac, s16 = audio[2 * i], audio[2 * i + 1]
        assert flac.dtype == np.uint8 and s16.dtype == np.int16 and len(s16) > 0
        y, r, frames = O.decode(flac.tobytes())
        assert r == (rate or 24000) and np.array_equal(y, s16), (rate, speed)
        assert int.from_bytes(flac[18:26].tobytes(), "big") & ((1 << 36) - 1) == 0   # streamed: total unknown
        assert all(n == 4096 or n % 16 == 0 for _, n, _, _ in frames[:-1])


def test_convert_of_a_one_shot_output(monkeypatch):
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    from faster_qwen3_tts import flac as F
    from faster_qwen3_tts.serving import to_pcm16
    m = _model()
    for rate in (8000, 24000):
        for speed in (1.0, 1.5):
            shot, sr = m.generate_custom_voice("hello there", "ryan", "English", speed=speed, sample_rate=rate, **GEN)
            s16 = np.frombuffer(to_pcm16(shot[0]), np.int16)
            data = _bytes(F.convert(_dev(s16), sr))
            y, r, _ = O.decode(data)
            assert r == rate and np.array_equal(y, s16), (rate, speed)
            assert int.from_bytes(data[18:26], "big") & ((1 << 36) - 1) == len(s16)   # one shot: total known
