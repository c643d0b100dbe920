"""GPU tests of the output-rate and encoding stage (csrc/fq3_resample.cu through faster_qwen3_tts/resample.py).

The kernel against the float64 oracle (oracle/resample_oracle.py) at every rate: each sample within the fp32 accumulation
bound gamma_{K+1} * sum |L h_j x_i| (K taps, the table's own rounding counted as one more).  The encodings bit for bit:
s16 is serving.to_pcm16 of the same kernel's f32 output, ulaw / alaw the G.711 of that s16, and the encode-only case
maps every s16 value exactly.  The output does not depend on the chunking of the input nor on which other streams share
the launch, bit for bit.  End to end on the synthetic model: every delivery at a rate is ``resample.convert`` of the same
request's 24 kHz output in one push, bit for bit, and the default launches nothing new."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import prompt_cases  # noqa: F401  (puts the package on sys.path)
from oracle import resample_oracle as O

pytestmark = pytest.mark.gpu

SR = 24000
RESAMPLED = (8000, 16000, 22050, 32000, 44100, 48000)
RATES = (8000, 16000, 22050, 24000, 32000, 44100, 48000)


def _dev(x):
    return torch.as_tensor(np.asarray(x, dtype=np.float32), device="cuda")


def _signals(rate, n=6000):
    """sines just inside the pass band and just above the lower Nyquist, white noise, impulses and step onsets"""
    ny = min(rate, SR) / 2
    t = np.arange(n) / SR
    rng = np.random.default_rng(rate)
    sig = {"passband": 0.7 * np.sin(2 * np.pi * 0.78 * ny * t + 0.3),
           "stopband": 0.7 * np.sin(2 * np.pi * min(1.04 * ny, 0.995 * SR / 2) * t),
           "noise": np.clip(0.3 * rng.standard_normal(n), -1, 1)}
    imp = np.zeros(n)
    imp[[0, 1, 777, 2000, 2001, n - 1]] = [0.9, -0.9, 1.0, 0.5, -1.0, 0.8]
    sig["impulses"] = imp
    step = np.zeros(n)
    step[1000:3000], step[4000:] = 0.8, -0.6
    sig["steps"] = step
    return {k: v.astype(np.float32) for k, v in sig.items()}


def _process_one(rate, encoding, x, pushes=None):
    """x pushed in the given lengths (one push by default), flushed with the last"""
    from faster_qwen3_tts import resample as R
    r = R.Resampler(rate, encoding, "cuda")
    pushes = pushes or [len(x)]
    parts, i = [], 0
    for k, n in enumerate(pushes):
        want = r.released(n, k == len(pushes) - 1)
        out = R.process([r], [x[i:i + n]], k == len(pushes) - 1)[0]
        assert out.numel() == want and out.dtype == R.DTYPES[encoding]
        parts.append(out.cpu())
        i += n
    r.close()
    return torch.cat(parts)


@pytest.mark.parametrize("rate", RESAMPLED)
def test_kernel_against_the_float64_oracle(rate):
    from faster_qwen3_tts import resample as R
    L, M, half = R.ratio(rate)
    K = 2 * half // L + 1
    u = 2.0 ** -24
    gamma = (K + 1) * u / (1 - (K + 1) * u)
    for name, x in _signals(rate).items():
        y = R.convert(_dev(x), rate).cpu().numpy().astype(np.float64)
        want = O.resample(x.astype(np.float64), rate)
        assert len(y) == len(want) == -(-len(x) * L // M)
        bound = gamma * O.magnitude(x, rate) + 1e-30
        err = np.abs(y - want)
        print(f"{rate} {name}: max err {err.max():.2e}, max err / bound {(err / bound).max():.3f}")
        assert (err <= bound).all(), (name, int(np.argmax(err / bound)))


@pytest.mark.parametrize("rate", RATES)
def test_encodings_bit_for_bit(rate):
    from faster_qwen3_tts.serving import to_pcm16
    x = _dev(np.concatenate([v for v in _signals(rate, 3000).values()]) * 1.3)   # some samples clip
    f32 = _process_one(rate, "f32", x).numpy() if rate != SR else x.cpu().numpy()
    s16 = _process_one(rate, "s16", x).numpy()
    assert s16.tobytes() == to_pcm16(f32)
    assert np.array_equal(_process_one(rate, "ulaw", x).numpy(), O.lin2ulaw(s16))
    assert np.array_equal(_process_one(rate, "alaw", x).numpy(), O.lin2alaw(s16))


def test_encode_only_maps_every_s16_value_exactly():
    s = np.arange(-32768, 32768, dtype=np.int16)
    x = _dev(s.astype(np.float32) / 32768)
    assert np.array_equal(_process_one(SR, "s16", x).numpy(), s)
    assert np.array_equal(_process_one(SR, "ulaw", x).numpy(), O.lin2ulaw(s))
    assert np.array_equal(_process_one(SR, "alaw", x).numpy(), O.lin2alaw(s))


@pytest.mark.parametrize("rate,encoding", [(r, "f32") for r in RESAMPLED] + [(8000, "ulaw"), (24000, "s16"),
                                                                               (44100, "alaw")])
def test_bit_identical_across_chunkings(rate, encoding):
    x = _dev(_signals(rate, 9000)["noise"])
    whole = _process_one(rate, encoding, x)
    rng = np.random.default_rng(rate)
    splits = []
    while sum(splits) < x.numel():
        splits.append(min(int(rng.integers(0, 2500)), x.numel() - sum(splits)))
    ones = [1] * 700 + [x.numel() - 700]
    for pushes in (splits, ones):
        assert torch.equal(_process_one(rate, encoding, x, pushes), whole)


def test_streams_in_one_launch_equal_each_alone():
    from faster_qwen3_tts import resample as R
    cfg = [(8000, "ulaw"), (48000, "f32"), (22050, "s16"), (24000, "alaw"), (44100, "f32"), (16000, "ulaw"),
           (32000, "s16"), (8000, "f32")]
    sigs = [_dev(_signals(r, 5000 + 911 * i)["noise"]) for i, (r, _) in enumerate(cfg)]
    alone = [_process_one(r, e, x) for (r, e), x in zip(cfg, sigs)]
    rs = [R.Resampler(r, e, "cuda") for r, e in cfg]
    parts = [[] for _ in cfg]
    pos = [0] * len(cfg)
    rng = np.random.default_rng(0)
    while any(p < x.numel() for p, x in zip(pos, sigs)):   # own push lengths (empty ones among them) and flush points
        live = [i for i in range(len(cfg)) if pos[i] < sigs[i].numel()]
        ns = [min(int(rng.integers(0, 2000)), sigs[i].numel() - pos[i]) for i in live]
        outs = R.process([rs[i] for i in live], [sigs[i][pos[i]:pos[i] + n] for i, n in zip(live, ns)],
                         [pos[i] + n == sigs[i].numel() for i, n in zip(live, ns)])
        for i, n, o in zip(live, ns, outs):
            assert o.data_ptr() % R.ALIGN == 0
            parts[i].append(o.cpu())
            pos[i] += n
    for i, r in enumerate(rs):
        r.close()
        assert torch.equal(torch.cat(parts[i]), alone[i]), cfg[i]


def test_bad_input_is_refused_before_any_launch():
    from faster_qwen3_tts import resample as R
    from faster_qwen3_tts.engine import load_library
    lib = load_library()
    h = C.c_void_p()
    for rate, enc in ((11025, 0), (96000, 1), (8000, 4), (8000, -1), (24000, 0)):
        assert lib.fq3_resample_create(0, rate, enc, C.byref(h)) == -1
    a, b = R.Resampler(8000, "ulaw", "cuda"), R.Resampler(48000, "f32", "cuda")
    x = torch.zeros(2000, device="cuda")
    out = torch.empty(16384, dtype=torch.uint8, device="cuda")
    lens, fl = (C.c_int64 * 2)(1000, 1000), (C.c_int32 * 2)(0, 0)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(handles, inp, outp, cap=16384):
        arr = (C.c_void_p * len(handles))(*[t._h for t in handles])
        return lib.fq3_resample_process(arr, len(handles), inp, lens, fl, outp, cap, stream)

    assert call([a, a], C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr())) == -1
    assert b"twice" in lib.fq3_resample_last_error()
    assert call([a, b], None, C.c_void_p(out.data_ptr())) == -1
    assert call([a, b], C.c_void_p(x.data_ptr() + 2), C.c_void_p(out.data_ptr())) == -1
    assert call([a, b], C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr() + 4)) == -1
    assert b"misaligned" in lib.fq3_resample_last_error()
    assert call([a, b], C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr()), cap=100) == -1
    assert b"smaller" in lib.fq3_resample_last_error()
    assert call([a, b], C.c_void_p(x.data_ptr()), None) == -1
    xs = _dev(_signals(8000, 3000)["noise"])
    assert torch.equal(R.process([a], [xs], True)[0].cpu(), _process_one(8000, "ulaw", xs))   # state untouched
    a = R.Resampler(8000, "ulaw", "cuda")
    with pytest.raises(ValueError, match="twice"):
        R.process([a, a], [x, x], False)
    with pytest.raises(ValueError, match="float32"):
        R.process([a], [x.double()], False)
    R.process([a], [x], True)
    with pytest.raises(ValueError, match="flushed"):
        R.process([a], [x], False)
    a.close()
    b.close()
    # a flushed handle from the pool starts a new stream
    c = R.Resampler(8000, "ulaw", "cuda")
    y = _dev(_signals(8000, 3000)["noise"])
    assert torch.equal(R.process([c], [y], True)[0].cpu(), _process_one(8000, "ulaw", y))
    c.close()


# ---- end to end on the synthetic model --------------------------------------------------------------------------------
def _model(max_batch=4):
    from faster_qwen3_tts import FasterQwen3TTS
    m = FasterQwen3TTS.from_synthetic("tiny", dtype=torch.bfloat16, max_seq_len=512, seed=5, max_batch=max_batch)
    m.predictor_graph.do_sample = False
    return m


def _converted(pcm, rate, encoding="f32"):
    from faster_qwen3_tts import resample as R
    return R.convert(_dev(pcm), rate, encoding).cpu().numpy()


GEN = dict(max_new_tokens=21, min_new_tokens=21, do_sample=False)


@pytest.mark.parametrize("codec_mode", ["window", "stateful"])
def test_streaming_and_one_shot_equal_the_conversion_of_24k(codec_mode, monkeypatch):
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    m = _model()
    m.streaming_codec = codec_mode
    kw = dict(ref_audio="ref.wav", ref_text="ref words", chunk_size=8, **GEN)
    for speed in (1.0, 1.5):
        base = np.concatenate([a for a, _, _ in m.generate_voice_clone_streaming("hello there", "English",
                                                                               speed=speed, **kw)])
        one = m.generate_custom_voice("hello there", "ryan", "English", speed=speed, **GEN)[0][0]
        for rate in (8000, 48000):
            items = list(m.generate_voice_clone_streaming("hello there", "English", speed=speed, sample_rate=rate, **kw))
            assert all(sr == rate for _, sr, _ in items) and items[-1][2]["chunk_steps"] == 0
            got = np.concatenate([a for a, _, _ in items])
            assert np.array_equal(got, _converted(base, rate)), (speed, rate)
            shot, sr = m.generate_custom_voice("hello there", "ryan", "English", speed=speed, sample_rate=rate, **GEN)
            assert sr == rate and np.array_equal(shot[0], _converted(one, rate)), (speed, rate)


def test_takes_and_batch_equal_the_conversion_of_24k(monkeypatch):
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    m = _model()
    gen = dict(max_new_tokens=30, min_new_tokens=2, temperature=0.9, top_k=50, top_p=1.0, do_sample=True,
               repetition_penalty=1.05)
    texts, spk, lang = ["one two three", "a second, longer request"], ["ryan", "ryan"], ["English"] * 2
    for speed in (1.0, 1.5):
        base, _, _ = m.generate_custom_voice_takes("several takes", "ryan", "English", n_takes=3, seeds=[1, 2, 3],
                                                   speed=speed, **gen)
        bbase, _ = m.generate_custom_voice_batch(texts, spk, lang, speed=speed, **GEN)
        for rate in (8000, 48000):
            got, sr, _ = m.generate_custom_voice_takes("several takes", "ryan", "English", n_takes=3, seeds=[1, 2, 3],
                                                       speed=speed, sample_rate=rate, **gen)
            assert sr == rate
            for b, g in zip(base, got):
                assert np.array_equal(g, _converted(b, rate)), (speed, rate)
            got, sr = m.generate_custom_voice_batch(texts, spk, lang, speed=speed, sample_rate=rate, **GEN)
            assert sr == rate
            for b, g in zip(bbase, got):
                assert np.array_equal(g, _converted(b, rate)), (speed, rate)


@pytest.mark.parametrize("codec_mode", ["window", "stateful"])
def test_continuous_batcher_tickets_at_their_own_rates(codec_mode, monkeypatch):
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    import time
    from faster_qwen3_tts.serving import batcher_for_model, voice_clone_request
    m = _model()
    m.streaming_codec = codec_mode
    texts = ["hello there general kenobi", "short one", "the quick brown fox jumps", "another request here"]
    outs = [(8000, "ulaw", 1.0), (48000, "f32", 1.5), (24000, "s16", 1.0), (16000, "alaw", 1.0)]
    b = batcher_for_model(m, chunk_size=8)
    try:
        def run(spec):
            tickets = []
            for i, (text, kw) in enumerate(zip(texts, spec)):
                tickets.append(b.submit(voice_clone_request(m, text, "English", "ref.wav", "ref words",
                                                            xvec_only=(i % 2 == 0)), **kw, **GEN))
                time.sleep(0.05)   # staggered arrivals
            return [t.audio() for t in tickets]
        base = run([dict(speed=s) for _, _, s in outs])
        got = run([dict(sample_rate=r, encoding=e, speed=s) for r, e, s in outs])
    finally:
        b.close()
    for g, a, (r, e, _) in zip(got, base, outs):
        assert np.array_equal(g, _converted(a, r, e)), (r, e)


def test_default_rate_launches_nothing_new(monkeypatch):
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    from faster_qwen3_tts import resample as R
    m = _model()
    calls = []
    real = R.process
    monkeypatch.setattr(R, "process", lambda *a, **k: calls.append(1) or real(*a, **k))

    def counts():
        torch.cuda.synchronize()
        return m.engine.launch_count, m.codec_launches()

    m.generate_custom_voice("hello there", "ryan", "English", **GEN)   # first call: warm-up launches
    c0 = counts()
    a = m.generate_custom_voice("hello there", "ryan", "English", **GEN)[0][0]
    c1 = counts()
    b = m.generate_custom_voice("hello there", "ryan", "English", sample_rate=24000, **GEN)[0][0]
    c2 = counts()
    assert np.array_equal(a, b) and calls == []
    assert (c2[0] - c1[0], c2[1] - c1[1]) == (c1[0] - c0[0], c1[1] - c0[1])
    items = list(m.generate_custom_voice_streaming("hello there", "ryan", "English", sample_rate=None, chunk_size=8,
                                                   **GEN))
    assert calls == [] and items


def test_speed_that_quantises_to_one_is_the_identity_in_every_delivery(monkeypatch):
    """speed 1.0004 passes the speed check and quantises to q = 1024: one-shot and takes return the speed-1 audio, at 24
    kHz and at a resampled rate"""
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    m = _model()
    gen = dict(max_new_tokens=30, min_new_tokens=2, temperature=0.9, top_k=50, top_p=1.0, do_sample=True,
               repetition_penalty=1.05)
    one = m.generate_custom_voice("hello there", "ryan", "English", **GEN)[0][0]
    takes, _, _ = m.generate_custom_voice_takes("several takes", "ryan", "English", n_takes=2, seeds=[1, 2], **gen)
    for rate in (None, 8000):
        want = one if rate is None else _converted(one, rate)
        shot, sr = m.generate_custom_voice("hello there", "ryan", "English", speed=1.0004, sample_rate=rate, **GEN)
        assert sr == (rate or 24000) and np.array_equal(shot[0], want), rate
        got, _, _ = m.generate_custom_voice_takes("several takes", "ryan", "English", n_takes=2, seeds=[1, 2],
                                                  speed=1.0004, sample_rate=rate, **gen)
        for b, g in zip(takes, got):
            assert np.array_equal(g, b if rate is None else _converted(b, rate)), rate
