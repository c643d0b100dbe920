"""GPU tests of long inputs (csrc/fq3_join.cu through faster_qwen3_tts/join.py, and segmented requests end to end).

The join kernel equals the numpy oracle (tests/join_oracle.py) bit for bit for random push sequences, several requests
in one launch, and pauses of 0, 1 and 2000 ms.  Through the synthetic model, for both codec policies and custom-voice,
voice-design and x-vector and ICL clone voices: the 24 kHz f32 audio of a split request equals the oracle's join of the
solo requests of its segments, each sampled with ``take_uniforms(segment_seed(seed, k))``.  With split=False no join is
created."""
import numpy as np
import pytest
import torch

from oracle import prompt_cases  # noqa: F401  (puts the package on sys.path)

import join_oracle as O

pytestmark = pytest.mark.gpu


def _pushes(rng, segs, joins):
    """random push sequences: per call, a random subset of (join, segment) with a random part of what is left"""
    left = [[0] * len(s) for s in segs]
    calls = []
    while True:
        call = []
        for j, (s, ps) in enumerate(zip(segs, left)):
            for k, x in enumerate(s):
                if ps[k] is None or rng.random() < 0.4:
                    continue
                n = int(rng.integers(0, len(x) - ps[k] + 1))
                end = ps[k] + n == len(x) and rng.random() < 0.6
                call.append((j, k, x[ps[k]:ps[k] + n], end))
                ps[k] = None if end else ps[k] + n
        calls.append(call)
        if all(p is None for ps in left for p in ps):
            return calls


@pytest.mark.parametrize("pause_ms", [0, 1, 2000])
def test_kernel_equals_oracle(pause_ms):
    from faster_qwen3_tts import join as J
    rng = np.random.default_rng(pause_ms)
    for trial in range(4):
        n_req = int(rng.integers(1, 6))
        segs = [[rng.standard_normal(int(rng.integers(0, 6000))).astype(np.float32)
                 for _ in range(int(rng.integers(1, 6)))] for _ in range(n_req)]
        joins = [J.Join(len(s), pause_ms, "cuda") for s in segs]
        got = [[] for _ in segs]
        for call in _pushes(rng, segs, joins):
            if not call:
                continue
            live = sorted({j for j, _, _, _ in call})
            outs = J.process([joins[j] for j in live],
                             [(joins[j], k, torch.from_numpy(x).cuda(), e) for j, k, x, e in call])
            for j, o in zip(live, outs):
                got[j].append(o.cpu().numpy())
        for j, s in enumerate(segs):
            assert joins[j].done
            y = np.concatenate(got[j]) if got[j] else np.zeros(0, np.float32)
            assert np.array_equal(y, O.join(s, pause_ms)), (trial, j)
            joins[j].close()
    # the one-call helper
    s = [rng.standard_normal(n).astype(np.float32) for n in (500, 90, 3000)]
    assert np.array_equal(J.join([torch.from_numpy(x).cuda() for x in s], pause_ms).cpu().numpy(),
                          O.join(s, pause_ms))


def test_kernel_refusals_before_launch():
    from faster_qwen3_tts import join as J
    j = J.Join(2, 0, "cuda")
    x = torch.zeros(10, device="cuda")
    with pytest.raises(ValueError):
        J.released([j], [(j, 2, x, False)])
    J.process([j], [(j, 0, x, True)])
    with pytest.raises(ValueError, match="ended"):
        J.released([j], [(j, 0, x, False)])
    with pytest.raises(ValueError, match="twice"):
        J.released([j, j], [(j, 1, x, False)])
    j.close()


GEN = dict(max_new_tokens=30, min_new_tokens=2, do_sample=True, temperature=0.9, top_k=50)
TEXT = "The first sentence is here, and it runs on. A second one follows it here. Third and last sentence now."


def _model():
    from faster_qwen3_tts import FasterQwen3TTS
    return FasterQwen3TTS.from_synthetic("tiny", dtype=torch.bfloat16, max_seq_len=512, seed=5, max_batch=8)


def _record_codes(b):
    """the codes every scheduler row emits, by row tag"""
    codes, step = {}, b.sched.step

    def recording(n):
        out = step(n)
        for rq, c in out:
            codes.setdefault(rq.tag, []).append(c.cpu())
        return out
    b.sched.step = recording
    return codes


def _solo(b, make, texts, seed):
    """each segment alone, with its documented uniforms, as an ordinary request on the same batcher"""
    from faster_qwen3_tts.model import take_uniforms
    from faster_qwen3_tts.segment import segment_seed
    out = []
    for k, s in enumerate(texts):
        t = b.submit(make(s), uniforms=take_uniforms(segment_seed(seed, k), GEN["max_new_tokens"], "cuda"), **GEN)
        out.append(t.audio())
    return out


@pytest.mark.parametrize("codec_mode", ["window", "stateful"])
@pytest.mark.parametrize("voice", ["custom", "design", "xvec", "icl"])
def test_split_request_equals_join_of_solo_segments(codec_mode, voice, monkeypatch):
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    from faster_qwen3_tts.segment import split_text
    from faster_qwen3_tts.serving import batcher_for_model, custom_voice_request, voice_clone_request
    m = _model()
    m.streaming_codec = codec_mode
    if voice == "custom":
        make = lambda s, **kw: custom_voice_request(m, s, "ryan", "English", **kw)
    elif voice == "design":
        make = lambda s, **kw: custom_voice_request(m, s, None, "English", instruct="a calm low voice", **kw)
    else:
        make = lambda s, **kw: voice_clone_request(m, s, "English", "ref.wav", "ref words", xvec_only=voice == "xvec",
                                                   **kw)
    texts = split_text(TEXT, 60)
    assert len(texts) == 3
    b = batcher_for_model(m, chunk_size=8)
    codes = _record_codes(b)
    try:
        t = b.submit(make(TEXT, split=True, max_segment_chars=60), split=True, pause_ms=40, seed=1234, **GEN)
        chunks = list(t)
        rows = sorted(codes)
        solo = _solo(b, make, texts, 1234)
    finally:
        b.close()
    # each row's codes equal those of its segment spoken alone with the documented seed
    solos = sorted(set(codes) - set(rows))
    assert len(rows) == len(solos) == 3
    for r, s in zip(rows, solos):
        assert torch.equal(torch.cat(codes[r]), torch.cat(codes[s]))
    audio = np.concatenate([c[0] for c in chunks])
    assert [c[2]["segment"] for c in chunks] == sorted(c[2]["segment"] for c in chunks)
    assert all(c[2]["n_segments"] == 3 for c in chunks) and chunks[-1][2]["is_final"]
    assert all(len(s) > 0 for s in solo)
    assert np.array_equal(audio, O.join(solo, 40))


def test_generate_split_one_shot_and_streaming(monkeypatch):
    """the public calls: one-shot split equals streaming split; split=False creates no join"""
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    from faster_qwen3_tts import join as J
    m = _model()
    m.streaming_codec = "stateful"
    shot, sr = m.generate_custom_voice(TEXT, "ryan", "English", split=True, max_segment_chars=60, pause_ms=10,
                                       seed=9, **GEN)
    chunks = list(m.generate_custom_voice_streaming(TEXT, "ryan", "English", split=True, max_segment_chars=60,
                                                    pause_ms=10, seed=9, chunk_size=12, **GEN))
    assert sr == 24000 and np.array_equal(shot[0], np.concatenate([c[0] for c in chunks]))
    calls = []
    monkeypatch.setattr(J.Join, "__init__", lambda *a, **k: calls.append(a) or (_ for _ in ()).throw(AssertionError))
    plain, _ = m.generate_custom_voice("Hello there.", "ryan", "English", **GEN)
    list(m.generate_custom_voice_streaming("Hello there.", "ryan", "English", **GEN))
    assert not calls and len(plain[0]) > 0


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _twin(pcm24, rate, pitch, gain_db, speed, encoding):
    """the one-shot stages applied to a joined 24 kHz f32 stream: convert(stretch(pcm24, q / 1024), R, enc, ...)"""
    from faster_qwen3_tts import resample as R
    from faster_qwen3_tts import tempo as T
    q = R.tempo_q(speed, pitch)
    return R.convert(T.stretch(_dev(pcm24), q / 1024), rate, encoding, pitch, gain_db).cpu().numpy()


# the post-codec chain on the joined stream: speed, pitch, 8 kHz mu-law, and FLAC at a pitch and gain
POST = [dict(speed=1.5, pitch=-3, sample_rate=8000, encoding="ulaw"),
        dict(speed=1.5, sample_rate=24000, encoding="f32"),
        dict(speed=1.5, pitch=-3, sample_rate=8000, encoding="flac", gain_db=-6)]


@pytest.mark.parametrize("codec_mode", ["window", "stateful"])
def test_post_codec_stages_run_once_on_the_joined_stream(codec_mode, monkeypatch):
    """a split request with a speed, pitch, rate, encoding or FLAC delivers the one-shot stages of its own 24 kHz f32
    join (the same request at the defaults): the stages are continuous across the boundaries"""
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    from oracle import flac_oracle as F
    from faster_qwen3_tts.serving import batcher_for_model, custom_voice_request
    m = _model()
    m.streaming_codec = codec_mode
    b = batcher_for_model(m, chunk_size=8)
    try:
        def run(**kw):
            return b.submit(custom_voice_request(m, TEXT, "ryan", "English", split=True, max_segment_chars=60),
                            split=True, pause_ms=40, seed=77, **kw, **GEN).audio()
        base = run()
        got = [run(**o) for o in POST]
    finally:
        b.close()
    assert base.dtype == np.float32 and len(base) > 0
    for g, o in zip(got, POST):
        p = (o["sample_rate"], o.get("pitch", 0), o.get("gain_db", 0), o["speed"])
        if o["encoding"] == "flac":
            dec = F.decode(bytes(g))
            samples, rate = dec[0], dec[1]
            assert rate == o["sample_rate"]
            assert np.array_equal(np.asarray(samples, dtype=np.int16), _twin(base, *p, "s16")), o
        else:
            assert np.array_equal(g, _twin(base, *p, o["encoding"])), o


def test_long_input_ends_with_its_last_segment(monkeypatch):
    """a 4096-character input at max_new_tokens=2048: every segment is a row that ends by itself (its EOS or its own
    2048 frames), and the request ends with its last segment, not at frame 2048 of the whole text"""
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    from faster_qwen3_tts import FasterQwen3TTS
    from faster_qwen3_tts.segment import split_text
    from faster_qwen3_tts.serving import batcher_for_model, custom_voice_request
    m = FasterQwen3TTS.from_synthetic("tiny", dtype=torch.bfloat16, max_seq_len=3072, seed=5, max_batch=16)
    m.streaming_codec = "stateful"
    text = ("This is one sentence of a long input, and it is spoken on a row of its own. " * 60)[:4096]
    n = len(split_text(text, 400))
    b = batcher_for_model(m, chunk_size=16)
    codes = _record_codes(b)
    try:
        t = b.submit(custom_voice_request(m, text, "ryan", "English", split=True), split=True, seed=3,
                     max_new_tokens=2048, min_new_tokens=2, do_sample=True)
        chunks = list(t)
    finally:
        b.close()
    frames = [sum(int(c.shape[0]) for c in codes[r]) for r in sorted(codes)]
    assert n >= 10 and len(frames) == n and all(0 < f <= 2048 for f in frames)
    assert chunks[-1][2]["is_final"] and chunks[-1][2]["segment"] == n - 1 and chunks[-1][2]["n_segments"] == n
    assert [c[2]["segment"] for c in chunks] == sorted(c[2]["segment"] for c in chunks)
    assert chunks[-1][2]["total_steps_so_far"] == sum(frames) > 2048
