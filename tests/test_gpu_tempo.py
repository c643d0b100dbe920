"""GPU tests of the speaking-rate stage (csrc/fq3_tempo.cu through faster_qwen3_tts/tempo.py).

The kernel against the float64 oracle (oracle/tempo_oracle.py) decision by decision: every p_k it chose is the oracle's
argmax or scores within 1e-5 relative of the maximum, and the oracle replaying the kernel's positions gives every sample
within 1e-6.  The output does not depend on the chunking of the input, nor on which other streams share the launch, bit
for bit.  End to end on the synthetic model: every delivery at speed s gives the GPU tempo of its speed-1 PCM in one push,
bit for bit, and speed 1 launches nothing new."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import prompt_cases  # noqa: F401  (puts the package on sys.path)
from oracle import tempo_oracle as O

pytestmark = pytest.mark.gpu

SR = 24000
SPEEDS = (0.25, 0.5, 0.8, 1.25, 1.5, 2.0, 4.0)


def _sines(n=SR):
    t = np.arange(n) / SR
    return 0.4 * np.sin(2 * np.pi * 110 * t) + 0.2 * np.sin(2 * np.pi * 220 * t + 1) + 0.1 * np.sin(2 * np.pi * 440 * t)


def _onsets(n=SR):
    x = np.zeros(n)
    rng = np.random.default_rng(3)
    for start in (3000, 9000, 15500, 21000):
        m = min(1500, n - start)
        x[start:start + m] = 0.6 * np.sin(2 * np.pi * 180 * np.arange(m) / SR) * np.exp(-np.arange(m) / 600)
        x[start:start + 40] += 0.3 * rng.standard_normal(40)
    return x


def _speech_like(n=SR, seed=7):
    """a glottal pulse train with a gliding f0 through three formant resonators, with noise bursts"""
    from scipy.signal import lfilter
    rng = np.random.default_rng(seed)
    f0 = 110 + 60 * np.sin(2 * np.pi * 1.3 * np.arange(n) / SR)
    phase = np.cumsum(f0 / SR)
    src = np.diff(np.floor(phase), prepend=0.0) * 1.0
    for fc, bw in ((700, 110), (1220, 120), (2600, 160)):
        r = np.exp(-np.pi * bw / SR)
        src = lfilter([1 - r], [1, -2 * r * np.cos(2 * np.pi * fc / SR), r * r], src)
    for s in rng.integers(0, n - 2400, 4):
        src[s:s + 2400] += 0.05 * rng.standard_normal(2400)
    return 0.5 * src / np.abs(src).max()


SIGNALS = {"sines": _sines, "onsets": _onsets, "speech": _speech_like}


def _dev(x):
    return torch.as_tensor(np.asarray(x, dtype=np.float32), device="cuda")


@pytest.mark.parametrize("speed", SPEEDS)
@pytest.mark.parametrize("signal", sorted(SIGNALS))
def test_kernel_against_the_float64_oracle(signal, speed):
    from faster_qwen3_tts import tempo as T
    x = SIGNALS[signal]().astype(np.float32)
    y, pk = T.stretch(_dev(x), speed, positions=True)
    y, pk = y.cpu().numpy(), pk.cpu().numpy()
    want, s = O.stretch(x.astype(np.float64), speed)
    assert len(y) == len(want) == T.out_len(len(x), T.quantize(speed))
    assert len(pk) == len(s.p) and pk[0] == 0
    replay_y, r = O.stretch(x.astype(np.float64), speed, forced=pk)
    worst = 0.0
    for k, (cand, c) in enumerate(r.scores, start=1):
        best = c.max()
        got = c[cand == pk[k]]
        assert got.size == 1, (k, pk[k])
        gap = (best - got[0]) / max(abs(best), 1e-30)
        worst = max(worst, gap)
        assert pk[k] == s.p[k] or gap <= 1e-5, (k, pk[k], gap)
    d = float(np.abs(y - replay_y).max()) if len(y) else 0.0
    print(f"{signal} x{speed}: {len(pk)} frames, {int((pk != np.asarray(s.p)).sum())} away from the float64 argmax, "
          f"worst relative score gap {worst:.2e}, max|y - replay| {d:.2e}")
    assert d <= 1e-6


@pytest.mark.parametrize("speed", SPEEDS)
def test_bit_identical_across_chunkings(speed):
    from faster_qwen3_tts import tempo as T
    x = _dev(_speech_like(12000, seed=int(speed * 10)))
    whole = T.stretch(x, speed).cpu()
    rng = np.random.default_rng(int(speed * 100))
    for mode in ("random", "ones"):
        t, parts, i = T.Tempo(speed, "cuda"), [], 0
        while i < x.numel():
            n = 1 if mode == "ones" and i < 2000 else int(rng.integers(1, 4000))
            n = min(n, x.numel() - i)
            parts.append(T.process([t], [x[i:i + n]], i + n == x.numel())[0].cpu())
            i += n
        t.close()
        assert torch.equal(torch.cat(parts), whole), mode


def test_streams_in_one_launch_equal_each_alone():
    from faster_qwen3_tts import tempo as T
    speeds = (0.5, 0.75, 1.25, 1.5, 2.0, 3.0, 0.25, 4.0)
    sigs = [_dev(_speech_like(6000 + 997 * i, seed=i)) for i in range(len(speeds))]
    alone = [T.stretch(x, s).cpu() for x, s in zip(sigs, speeds)]
    tempos = [T.Tempo(s, "cuda") for s in speeds]
    parts = [[] for _ in speeds]
    rng = np.random.default_rng(0)
    pos = [0] * len(speeds)
    while any(p < x.numel() for p, x in zip(pos, sigs)):   # each stream its own push lengths and flush point
        live = [i for i in range(len(speeds)) if pos[i] < sigs[i].numel()]
        ns = [min(int(rng.integers(1, 3000)), sigs[i].numel() - pos[i]) for i in live]
        outs = T.process([tempos[i] for i in live], [sigs[i][pos[i]:pos[i] + n] for i, n in zip(live, ns)],
                         [pos[i] + n == sigs[i].numel() for i, n in zip(live, ns)])
        for i, n, o in zip(live, ns, outs):
            parts[i].append(o.cpu())
            pos[i] += n
    for i, t in enumerate(tempos):
        t.close()
        assert torch.equal(torch.cat(parts[i]), alone[i]), speeds[i]


def test_bad_input_is_refused_before_any_launch():
    from faster_qwen3_tts import tempo as T
    from faster_qwen3_tts.engine import load_library
    lib = load_library()
    h = C.c_void_p()
    for bad in (0.2, 4.5, 1.0):
        assert lib.fq3_tempo_create(0, C.c_double(bad), C.byref(h)) == -1
    a, b = T.Tempo(1.5, "cuda"), T.Tempo(0.5, "cuda")
    x = torch.zeros(2000, device="cuda")
    out = torch.empty(8000, device="cuda")
    lens, fl = (C.c_int64 * 2)(1000, 1000), (C.c_int32 * 2)(0, 0)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(handles, inp, outp, cap=8000):
        arr = (C.c_void_p * len(handles))(*[t._h for t in handles])
        return lib.fq3_tempo_process(arr, len(handles), inp, lens, fl, outp, cap, None, 0, stream)

    assert call([a, a], C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr())) == -1
    assert b"twice" in lib.fq3_tempo_last_error()
    assert call([a, b], None, C.c_void_p(out.data_ptr())) == -1
    assert call([a, b], C.c_void_p(x.data_ptr() + 2), C.c_void_p(out.data_ptr())) == -1
    assert b"misaligned" in lib.fq3_tempo_last_error()
    assert call([a, b], C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr()), cap=10) == -1
    with pytest.raises(ValueError, match="twice"):
        T.process([a, a], [x, x], False)
    T.process([a], [x], True)
    with pytest.raises(ValueError, match="flushed"):
        T.process([a], [x], False)
    a.close()
    b.close()


# ---- end to end on the synthetic model --------------------------------------------------------------------------------
def _model(max_batch=4):
    from faster_qwen3_tts import FasterQwen3TTS
    m = FasterQwen3TTS.from_synthetic("tiny", dtype=torch.bfloat16, max_seq_len=512, seed=5, max_batch=max_batch)
    m.predictor_graph.do_sample = False
    return m


def _stretched(pcm, speed):
    from faster_qwen3_tts import tempo as T
    return T.stretch(_dev(pcm), speed).cpu().numpy()


GEN = dict(max_new_tokens=21, min_new_tokens=21, do_sample=False)


@pytest.mark.parametrize("codec_mode", ["window", "stateful"])
def test_streaming_and_one_shot_equal_the_tempo_of_speed_one(codec_mode, monkeypatch):
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    m = _model()
    m.streaming_codec = codec_mode
    kw = dict(ref_audio="ref.wav", ref_text="ref words", chunk_size=8, **GEN)
    base = np.concatenate([a for a, _, _ in m.generate_voice_clone_streaming("hello there", "English", **kw)])
    one = m.generate_custom_voice("hello there", "ryan", "English", **GEN)[0][0]
    for speed in (0.75, 1.5, 2.0):
        got = [a for a, _, _ in m.generate_voice_clone_streaming("hello there", "English", speed=speed, **kw)]
        assert np.array_equal(np.concatenate(got), _stretched(base, speed)), speed
        shot = m.generate_custom_voice("hello there", "ryan", "English", speed=speed, **GEN)[0][0]
        assert np.array_equal(shot, _stretched(one, speed)), speed


def test_takes_and_batch_equal_the_tempo_of_speed_one(monkeypatch):
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    m = _model()
    gen = dict(max_new_tokens=30, min_new_tokens=2, temperature=0.9, top_k=50, top_p=1.0, do_sample=True,
               repetition_penalty=1.05)
    base, _, _ = m.generate_custom_voice_takes("several takes", "ryan", "English", n_takes=3, seeds=[1, 2, 3], **gen)
    got, _, _ = m.generate_custom_voice_takes("several takes", "ryan", "English", n_takes=3, seeds=[1, 2, 3], speed=1.5,
                                              **gen)
    for b, g in zip(base, got):
        assert np.array_equal(g, _stretched(b, 1.5))
    texts, spk, lang = ["one two three", "a second, longer request"], ["ryan", "ryan"], ["English"] * 2
    base, _ = m.generate_custom_voice_batch(texts, spk, lang, **GEN)
    got, _ = m.generate_custom_voice_batch(texts, spk, lang, speed=0.75, **GEN)
    for b, g in zip(base, got):
        assert np.array_equal(g, _stretched(b, 0.75))


@pytest.mark.parametrize("codec_mode", ["window", "stateful"])
def test_continuous_batcher_tickets_at_their_own_speeds(codec_mode, monkeypatch):
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    import time
    from faster_qwen3_tts.serving import batcher_for_model, voice_clone_request
    m = _model()
    m.streaming_codec = codec_mode
    texts = ["hello there general kenobi", "short one", "the quick brown fox jumps", "another request here"]
    speeds = (1.0, 0.75, 1.5, 2.0)
    alone = []
    for i, text in enumerate(texts):
        parts = [p for p, _, _ in m.generate_voice_clone_streaming(text, "English", ref_audio="ref.wav",
                                                                    ref_text="ref words", chunk_size=8,
                                                                    xvec_only=(i % 2 == 0), **GEN)]
        alone.append(np.concatenate(parts))
    b = batcher_for_model(m, chunk_size=8)
    try:
        tickets = []
        for i, (text, s) in enumerate(zip(texts, speeds)):
            tickets.append(b.submit(voice_clone_request(m, text, "English", "ref.wav", "ref words",
                                                        xvec_only=(i % 2 == 0)), speed=s, **GEN))
            time.sleep(0.05)   # staggered arrivals
        got = [t.audio() for t in tickets]
    finally:
        b.close()
    assert np.array_equal(got[0], alone[0])
    for g, a, s in zip(got[1:], alone[1:], speeds[1:]):
        assert np.array_equal(g, _stretched(a, s)), s


def test_speed_one_launches_nothing_new(monkeypatch):
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    from faster_qwen3_tts import tempo as T
    m = _model()
    calls = []
    real = T.process
    monkeypatch.setattr(T, "process", lambda *a, **k: calls.append(1) or real(*a, **k))

    def counts():
        torch.cuda.synchronize()
        return m.engine.launch_count, m.codec_launches()

    m.generate_custom_voice("hello there", "ryan", "English", **GEN)   # first call: warm-up launches
    c0 = counts()
    a = m.generate_custom_voice("hello there", "ryan", "English", **GEN)[0][0]
    c1 = counts()
    b = m.generate_custom_voice("hello there", "ryan", "English", speed=1.0, **GEN)[0][0]
    c2 = counts()
    assert np.array_equal(a, b) and calls == []
    assert (c2[0] - c1[0], c2[1] - c1[1]) == (c1[0] - c0[0], c1[1] - c0[1])
    list(m.generate_custom_voice_streaming("hello there", "ryan", "English", speed=1.0, chunk_size=8, **GEN))
    assert calls == []
