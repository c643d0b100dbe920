"""GPU tests of pitch and gain (csrc/fq3_resample.cu at a pitch rho, through faster_qwen3_tts/resample.py).

The kernel against the float64 oracle (tests/pitch_oracle.py) at every rate and rho in {128, 181, 256, 383, 509, 512},
the largest tables among them: each sample within the fp32 accumulation bound gamma_{K+1} * sum |L h_j x_i|.  The gain is
one fp32 multiply of that sum, so a gained output equals the ungained one times g bit for bit, and the encodings are
to_pcm16 / G.711 of the kernel's own gained f32, clipping included.  Chunkings and shared launches change no bit.  The
phase tables a device holds stay bounded however many pitches are used.  End to end on the synthetic model, every
delivery at a pitch and gain is ``resample.convert(tempo.stretch(pcm24, q / 1024), R, enc, pitch, gain_db)`` of its own
24 kHz speed-1 output, bit for bit, and pitch 0 at 0 dB creates and launches nothing new."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import prompt_cases  # noqa: F401  (puts the package on sys.path)
from oracle import resample_oracle as O
import pitch_oracle as P

pytestmark = pytest.mark.gpu

RATES = (8000, 16000, 22050, 24000, 32000, 44100, 48000)
RHOS = (128, 181, 256, 383, 509, 512)
PITCH_OF = {128: -12, 181: -6, 256: 0, 383: 6.977, 509: 11.9, 512: 12}   # semitones whose rho is the key


def _dev(x):
    return torch.as_tensor(np.asarray(x, dtype=np.float32), device="cuda")


def _signal(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 24000
    x = 0.4 * np.sin(2 * np.pi * 1234.5 * t) + np.clip(0.25 * rng.standard_normal(n), -1, 1)
    x[[0, 1, n // 3, n - 1]] = [0.9, -0.9, 1.0, -1.0]
    return x.astype(np.float32)


def _process(rate, encoding, x, pitch=0, gain_db=0, pushes=None):
    from faster_qwen3_tts import resample as R
    r = R.Resampler(rate, encoding, "cuda", pitch, gain_db)
    pushes = pushes or [len(x)]
    parts, i = [], 0
    for k, n in enumerate(pushes):
        fin = k == len(pushes) - 1
        want = r.released(n, fin)
        out = R.process([r], [x[i:i + n]], fin)[0]
        assert out.numel() == want and out.dtype == R.DTYPES[encoding]
        parts.append(out.cpu())
        i += n
    r.close()
    return torch.cat(parts)


def test_pitch_keys_map_to_their_rho():
    from faster_qwen3_tts import resample as R
    assert {rho: R.pitch_rho(p) for rho, p in PITCH_OF.items()} == {rho: rho for rho in RHOS}


@pytest.mark.parametrize("rho", RHOS)
@pytest.mark.parametrize("rate", RATES)
def test_kernel_against_the_float64_oracle(rate, rho):
    from faster_qwen3_tts import resample as R
    L, M, half = R.ratio(rate, rho)
    K = 2 * half // L + 1
    u = 2.0 ** -24
    gamma = (K + 1) * u / (1 - (K + 1) * u)
    x = _signal(4000, rate + rho)
    y = _process(rate, "f32", _dev(x), PITCH_OF[rho]).numpy().astype(np.float64) if (rate, rho) != (24000, 256) \
        else x.astype(np.float64)
    want = P.resample(x.astype(np.float64), rate, rho)
    assert len(y) == len(want) == -(-len(x) * L // M)
    bound = gamma * P.magnitude(x, rate, rho) + 1e-30
    err = np.abs(y - want)
    print(f"{rate} rho {rho}: L {L} M {M} taps {2 * half + 1}, max err / bound {(err / bound).max():.3f}")
    assert (err <= bound).all(), int(np.argmax(err / bound))


@pytest.mark.parametrize("rate,rho", [(8000, 171), (24000, 256), (22050, 509), (48000, 323), (48000, 512)])
def test_gain_and_encodings_bit_for_bit(rate, rho):
    """g * (the ungained f32) in fp32, and s16 / G.711 of that, at gains that clip (+16 dB) and that nearly mute"""
    from faster_qwen3_tts import resample as R
    from faster_qwen3_tts.serving import to_pcm16
    pitch = {171: -7, 256: 0, 509: 11.9, 323: 4, 512: 12}[rho]
    x = _dev(_signal(5000, rate) * 0.9)
    plain = _process(rate, "f32", x, pitch).numpy() if (rate, rho) != (24000, 256) else x.cpu().numpy()
    for db in (0, -6, 16, -96, 3.3):
        g = np.float32(R.gain_of(db))
        f32 = _process(rate, "f32", x, pitch, db).numpy() if (rate, rho, db) != (24000, 256, 0) else plain
        assert np.array_equal(f32, plain * g), db
        s16 = _process(rate, "s16", x, pitch, db).numpy()
        assert s16.tobytes() == to_pcm16(f32), db
        assert np.array_equal(_process(rate, "ulaw", x, pitch, db).numpy(), O.lin2ulaw(s16))
        assert np.array_equal(_process(rate, "alaw", x, pitch, db).numpy(), O.lin2alaw(s16))
        if db == 16:
            assert (np.abs(s16.astype(np.int32)) >= 32767).any()   # some samples clip


@pytest.mark.parametrize("rate,pitch,encoding", [(8000, 12, "ulaw"), (22050, 11.9, "f32"), (44100, -6, "s16"),
                                                 (24000, 7, "f32"), (16000, -12, "alaw")])
def test_bit_identical_across_chunkings(rate, pitch, encoding):
    x = _dev(_signal(9000, rate))
    whole = _process(rate, encoding, x, pitch, -3)
    rng = np.random.default_rng(rate)
    splits = []
    while sum(splits) < x.numel():
        splits.append(min(int(rng.integers(0, 2500)), x.numel() - sum(splits)))
    ones = [1] * 700 + [x.numel() - 700]
    for pushes in (splits, ones):
        assert torch.equal(_process(rate, encoding, x, pitch, -3, pushes), whole)


def test_mixed_streams_in_one_launch_equal_each_alone():
    """rates, pitches, gains and encodings in one launch; the plain streams among them equal today's convert"""
    from faster_qwen3_tts import resample as R
    cfg = [(8000, 12, 0, "ulaw"), (48000, 0, 0, "f32"), (22050, 11.9, -6, "s16"), (24000, 0, 0, "alaw"),
           (44100, -5, 6, "f32"), (16000, 0, -20, "ulaw"), (32000, 3, 0, "s16"), (8000, 0, 0, "f32"),
           (24000, 0, -6, "f32"), (48000, 12, 0, "f32")]
    sigs = [_dev(_signal(5000 + 911 * i, i)) for i in range(len(cfg))]
    alone = [_process(r, e, x, p, g) for (r, p, g, e), x in zip(cfg, sigs)]
    for (r, p, g, e), x, a in zip(cfg, sigs, alone):
        if (p, g) == (0, 0):
            assert torch.equal(a, R.convert(x, r, e).cpu())
    rs = [R.Resampler(r, e, "cuda", p, g) for r, p, g, e in cfg]
    parts = [[] for _ in cfg]
    pos = [0] * len(cfg)
    rng = np.random.default_rng(0)
    while any(p < x.numel() for p, x in zip(pos, sigs)):
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
    for rate, rho, enc in ((11025, 256, 0), (8000, 127, 1), (8000, 513, 1), (8000, 300, 4), (48000, 0, 0)):
        assert lib.fq3_resample_create_pitch(0, rate, rho, enc, C.byref(h)) == -1
    assert lib.fq3_resample_create(0, 24000, 0, C.byref(h)) == -1   # the plain entry point still refuses the identity
    r = R.Resampler(8000, "f32", "cuda", 5)
    for g in (float("nan"), float("inf"), -1.0):
        assert lib.fq3_resample_set_gain(r._h, C.c_float(g)) == -1
    x = _dev(_signal(3000, 1))
    assert torch.equal(R.process([r], [x], True)[0].cpu(), _process(8000, "f32", x, 5))   # gain untouched
    r.close()
    for kw in (dict(pitch=13), dict(gain_db=20), dict(pitch=float("nan"))):
        with pytest.raises(ValueError):
            R.convert(x, 8000, "f32", **kw)


def test_table_memory_stays_bounded_over_many_pitches():
    """20 distinct pitched tables at 22.05 kHz come and go: what stays is at most the pools' and the idle cache's"""
    from faster_qwen3_tts import resample as R
    from faster_qwen3_tts.engine import load_library
    lib = load_library()
    dev = torch.cuda.current_device()
    x = _dev(_signal(2000, 3))
    R.convert(x, 22050, "s16")   # the plain table, kept for the process
    base = lib.fq3_resample_table_bytes(dev)
    rhos = list(range(300, 320))
    sizes = {}
    for rho in rhos:
        pitch = 12 * np.log2(rho / 256)
        assert R.pitch_rho(pitch) == rho
        L, M, half = R.ratio(22050, rho)
        sizes[rho] = L * (2 * half // L + 1) * 4
        R.convert(x, 22050, "s16", pitch)
        assert lib.fq3_resample_table_bytes(dev) - base <= sum(sorted(sizes.values())[-2 * R.TABLE_CACHE:])
    held = lib.fq3_resample_table_bytes(dev) - base
    print(f"tables of 20 pitches: {sum(sizes.values())} B, held afterwards: {held} B")
    assert held <= sum(sorted(sizes.values())[-2 * R.TABLE_CACHE:]) < sum(sizes.values())
    assert len([k for k in R.Resampler._pool if k[2] != 256]) <= R.TABLE_CACHE


# ---- end to end on the synthetic model --------------------------------------------------------------------------------
def _model(max_batch=4):
    from faster_qwen3_tts import FasterQwen3TTS
    m = FasterQwen3TTS.from_synthetic("tiny", dtype=torch.bfloat16, max_seq_len=512, seed=5, max_batch=max_batch)
    m.predictor_graph.do_sample = False
    return m


def _twin(pcm24, rate, pitch, gain_db, speed=1.0, encoding="f32"):
    """convert(stretch(pcm24, q / 1024), R, enc, pitch, gain_db) of a 24 kHz speed-1 output"""
    from faster_qwen3_tts import resample as R
    from faster_qwen3_tts import tempo as T
    q = R.tempo_q(speed, pitch)
    return R.convert(T.stretch(_dev(pcm24), q / 1024), rate, encoding, pitch, gain_db).cpu().numpy()


GEN = dict(max_new_tokens=21, min_new_tokens=21, do_sample=False)
# (pitch, speed, rate, gain_db): a stretch and a tape-speed resample (q = 1024 at +7 and 1.5), two rates and gains
CASES = [(-5, 1.0, 8000, 0), (7, 1.5, 24000, -6), (-5, 1.5, 24000, 0), (7, 1.0, 8000, -6)]


@pytest.mark.parametrize("codec_mode", ["window", "stateful"])
def test_streaming_and_one_shot_equal_the_twin_of_24k(codec_mode, monkeypatch):
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    m = _model()
    m.streaming_codec = codec_mode
    kw = dict(ref_audio="ref.wav", ref_text="ref words", chunk_size=8, **GEN)
    base = np.concatenate([a for a, _, _ in m.generate_voice_clone_streaming("hello there", "English", **kw)])
    one = m.generate_custom_voice("hello there", "ryan", "English", **GEN)[0][0]
    for pitch, speed, rate, db in CASES:
        p = dict(pitch=pitch, speed=speed, sample_rate=rate, gain_db=db)
        items = list(m.generate_voice_clone_streaming("hello there", "English", **p, **kw))
        assert all(sr == rate for _, sr, _ in items) and items[-1][2]["chunk_steps"] == 0
        assert np.array_equal(np.concatenate([a for a, _, _ in items]), _twin(base, rate, pitch, db, speed)), p
        shot, sr = m.generate_custom_voice("hello there", "ryan", "English", **p, **GEN)
        assert sr == rate and np.array_equal(shot[0], _twin(one, rate, pitch, db, speed)), p


def test_takes_and_batch_equal_the_twin_of_24k(monkeypatch):
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    m = _model()
    gen = dict(max_new_tokens=30, min_new_tokens=2, temperature=0.9, top_k=50, top_p=1.0, do_sample=True,
               repetition_penalty=1.05)
    texts, spk, lang = ["one two three", "a second, longer request"], ["ryan", "ryan"], ["English"] * 2
    base, _, _ = m.generate_custom_voice_takes("several takes", "ryan", "English", n_takes=3, seeds=[1, 2, 3], **gen)
    bbase, _ = m.generate_custom_voice_batch(texts, spk, lang, **GEN)
    for pitch, speed, rate, db in CASES[:2]:
        p = dict(pitch=pitch, speed=speed, sample_rate=rate, gain_db=db)
        got, sr, _ = m.generate_custom_voice_takes("several takes", "ryan", "English", n_takes=3, seeds=[1, 2, 3],
                                                   **p, **gen)
        assert sr == rate
        for b, g in zip(base, got):
            assert np.array_equal(g, _twin(b, rate, pitch, db, speed)), p
        got, sr = m.generate_custom_voice_batch(texts, spk, lang, **p, **GEN)
        assert sr == rate
        for b, g in zip(bbase, got):
            assert np.array_equal(g, _twin(b, rate, pitch, db, speed)), p


@pytest.mark.parametrize("codec_mode", ["window", "stateful"])
def test_continuous_batcher_tickets_and_flac(codec_mode, monkeypatch):
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    import time
    from oracle import flac_oracle as F
    from faster_qwen3_tts.serving import batcher_for_model, voice_clone_request
    m = _model()
    m.streaming_codec = codec_mode
    texts = ["hello there general kenobi", "short one", "the quick brown fox jumps", "another request here"]
    outs = [dict(sample_rate=8000, encoding="ulaw", pitch=-5, speed=1.0),
            dict(sample_rate=24000, encoding="f32", pitch=7, speed=1.5, gain_db=-6),
            dict(sample_rate=24000, encoding="s16", pitch=7, gain_db=-6),
            dict(sample_rate=8000, encoding="flac", pitch=-5, speed=1.5)]
    b = batcher_for_model(m, chunk_size=8)
    try:
        def run(spec):
            tickets = []
            for i, (text, kw) in enumerate(zip(texts, spec)):
                tickets.append(b.submit(voice_clone_request(m, text, "English", "ref.wav", "ref words",
                                                            xvec_only=(i % 2 == 0)), **kw, **GEN))
                time.sleep(0.05)   # staggered arrivals
            return [t.audio() for t in tickets]
        base = run([{}] * 4)
        got = run(outs)
        twin = run([dict(o, encoding="s16") for o in outs])   # the flac ticket's s16 twin
    finally:
        b.close()
    for g, a, o in zip(got, base, outs):
        if o["encoding"] == "flac":
            continue
        want = _twin(a, o["sample_rate"], o["pitch"], o.get("gain_db", 0), o.get("speed", 1.0), o["encoding"])
        assert np.array_equal(g, want), o
    dec = F.decode(bytes(got[3]))
    samples = dec[0] if isinstance(dec, tuple) else dec
    s16 = _twin(base[3], 8000, -5, 0, 1.5, "s16")
    assert np.array_equal(np.asarray(samples, dtype=np.int16), twin[3]) and np.array_equal(twin[3], s16)


def test_pitch_zero_and_zero_db_create_and_launch_nothing_new(monkeypatch):
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    from faster_qwen3_tts import resample as R
    from faster_qwen3_tts import tempo as T
    m = _model()
    calls = []
    for mod, name in ((R, "process"), (T, "process"), (R, "Resampler"), (T, "Tempo")):
        real = getattr(mod, name)
        monkeypatch.setattr(mod, name, (lambda real, name: lambda *a, **k: calls.append(name) or real(*a, **k))(real,
                                                                                                                 name))

    def counts():
        torch.cuda.synchronize()
        return m.engine.launch_count, m.codec_launches()

    m.generate_custom_voice("hello there", "ryan", "English", **GEN)   # first call: warm-up launches
    c0 = counts()
    a = m.generate_custom_voice("hello there", "ryan", "English", **GEN)[0][0]
    c1 = counts()
    b = m.generate_custom_voice("hello there", "ryan", "English", pitch=0, gain_db=0.0, **GEN)[0][0]
    c2 = counts()
    assert np.array_equal(a, b) and calls == []
    assert (c2[0] - c1[0], c2[1] - c1[1]) == (c1[0] - c0[0], c1[1] - c0[1])
    items = list(m.generate_custom_voice_streaming("hello there", "ryan", "English", pitch=0.0, gain_db=-0.0,
                                                   chunk_size=8, **GEN))
    assert calls == [] and items
