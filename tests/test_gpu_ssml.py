"""GPU tests of SSML input (faster_qwen3_tts/ssml.py) and the join's pause per boundary (csrc/fq3_join.cu).

The join kernel with a pause plan equals ``join_pauses_oracle.join_pauses`` bit for bit for random push sequences and
plans drawn from 0 - 10 000 ms, leading and trailing silence included; the uniform plan gives the bits of
``fq3_join_create``.
Through the synthetic model, for both codec policies: a document with two clone voices, a custom speaker, nested
prosody and breaks speaks every segment as that segment alone in its voice, and its audio is the oracle's join of the
solo segments after each one's own tempo and resampler; request-level stages apply once to that join."""
import numpy as np
import pytest
import torch

from oracle import prompt_cases  # noqa: F401  (puts the package on sys.path)

import join_oracle as O
from join_pauses_oracle import join_pauses

pytestmark = pytest.mark.gpu


def _calls(rng, segs):
    """random push sequences: per call, a random subset of (join, segment) with a random part of what is left"""
    left = [[0] * len(s) for s in segs]
    calls = []
    while any(p is not None for ps in left for p in ps):
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
    return calls


def _run(joins, calls, J):
    got = [[] for _ in joins]
    for call in calls:
        if not call:
            continue
        live = sorted({j for j, _, _, _ in call})
        counts = J.released([joins[j] for j in live], [(joins[j], k, torch.from_numpy(x).cuda(), e)
                                                        for j, k, x, e in call])
        outs = J.process([joins[j] for j in live], [(joins[j], k, torch.from_numpy(x).cuda(), e) for j, k, x, e in call])
        for j, o, n in zip(live, outs, counts):
            assert o.numel() == n
            got[j].append(o.cpu().numpy())
    return [np.concatenate(g) if g else np.zeros(0, np.float32) for g in got]


def test_kernel_with_pause_plans_equals_oracle():
    from faster_qwen3_tts import join as J
    rng = np.random.default_rng(7)
    for trial in range(6):
        n_req = int(rng.integers(1, 5))
        segs = [[rng.standard_normal(int(rng.integers(0, 6000))).astype(np.float32)
                 for _ in range(int(rng.integers(1, 6)))] for _ in range(n_req)]
        plans = [[int(rng.choice([0, 1, int(rng.integers(0, 10001)), 10000])) for _ in range(len(s) + 1)] for s in segs]
        joins = [J.Join(len(s), 0, "cuda", pauses=p) for s, p in zip(segs, plans)]
        got = _run(joins, _calls(rng, segs), J)
        for j, (s, p) in enumerate(zip(segs, plans)):
            assert joins[j].done
            assert np.array_equal(got[j], join_pauses(s, p)), (trial, j, p)
            joins[j].close()
    # the one-call helper, with leading and trailing silence
    s = [rng.standard_normal(n).astype(np.float32) for n in (500, 90, 3000)]
    plan = [200, 0, 10000, 500]
    assert np.array_equal(J.join([torch.from_numpy(x).cuda() for x in s], pauses=plan).cpu().numpy(),
                          join_pauses(s, plan))


@pytest.mark.parametrize("pause_ms", [0, 1, 2000])
def test_uniform_plan_gives_the_bits_of_pause_ms(pause_ms):
    """fq3_join_create(pause_ms) and fq3_join_create_pauses([0, P, ..., P, 0]) release the same samples per call"""
    from faster_qwen3_tts import join as J
    rng = np.random.default_rng(pause_ms + 100)
    for trial in range(3):
        segs = [[rng.standard_normal(int(rng.integers(0, 5000))).astype(np.float32)
                 for _ in range(int(rng.integers(1, 6)))]]
        S = len(segs[0])
        calls = _calls(rng, segs)
        a = _run([J.Join(S, pause_ms, "cuda")], calls, J)[0]
        b = _run([J.Join(S, 0, "cuda", pauses=[0] + [pause_ms] * (S - 1) + [0])], calls, J)[0]
        assert np.array_equal(a, b) and np.array_equal(a, O.join(segs[0], pause_ms))


def test_pause_plan_refusals():
    from faster_qwen3_tts import join as J
    with pytest.raises(ValueError):
        J.Join(2, 0, "cuda", pauses=[0, 10001, 0])
    with pytest.raises(ValueError):
        J.Join(2, 0, "cuda", pauses=[0, 0])
    with pytest.raises(ValueError):
        J.Join(2, 0, "cuda", pauses=[0, -1, 0])


GEN = dict(max_new_tokens=30, min_new_tokens=2, do_sample=True, temperature=0.9, top_k=50)
VOICES = {"x": {"ref_audio": "ref.wav", "ref_text": "ref words", "xvec_only": True, "language": "English"},
          "i": {"ref_audio": "ref.wav", "ref_text": "ref words", "language": "English"},
          "c": {"speaker": "ryan", "language": "English"}}
DOC = ("<speak version='1.0'><break time='200ms'/>"
       "<voice name='x'>The first voice speaks this sentence here.</voice><break time='0ms'/>"
       "<voice name='i'>The second voice, cloned with its reference, answers.</voice><break time='250ms'/>"
       "<voice name='c'><prosody rate='1.5'>A custom speaker talks faster <prosody pitch='-3st'>and lower "
       "<prosody volume='-6dB'>and softer at the end.</prosody></prosody></prosody></voice><break time='1.5s'/>"
       "<voice name='x'>Back to the first voice to close.</voice><break time='500ms'/></speak>")
PAUSE = 40


def _model():
    from faster_qwen3_tts import FasterQwen3TTS
    return FasterQwen3TTS.from_synthetic("tiny", dtype=torch.bfloat16, max_seq_len=512, seed=5, max_batch=8)


def _record_codes(b):
    codes, step = {}, b.sched.step

    def recording(n):
        out = step(n)
        for rq, c in out:
            codes.setdefault(rq.tag, []).append(c.cpu())
        return out
    b.sched.step = recording
    return codes


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _stages(pcm24, speed, pitch, gain_db, rate=24000, encoding="f32"):
    """the one-shot stages: convert(stretch(pcm, q / 1024), rate, encoding, pitch, gain_db)"""
    from faster_qwen3_tts import resample as R
    from faster_qwen3_tts import tempo as T
    q = R.tempo_q(speed, pitch)
    x = _dev(pcm24)
    if q != 1024:
        x = T.stretch(x, q / 1024)
    return R.convert(x, rate, encoding, pitch, gain_db).cpu().numpy()


POST = [dict(speed=1.25, sample_rate=8000, encoding="ulaw"),
        dict(speed=1.25, sample_rate=24000, encoding="flac")]


@pytest.mark.parametrize("codec_mode", ["window", "stateful"])
def test_document_equals_join_of_solo_segments(codec_mode, monkeypatch):
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    from oracle import flac_oracle as F
    from faster_qwen3_tts.model import take_uniforms
    from faster_qwen3_tts.segment import segment_seed
    from faster_qwen3_tts.serving import batcher_for_model, ssml_request
    from faster_qwen3_tts.ssml import parse, voice_request
    m = _model()
    m.streaming_codec = codec_mode
    doc = parse(DOC, VOICES)
    assert [(s.voice, s.speed, s.pitch, s.gain_db) for s in doc.spans] == [
        ("x", 1, 0, 0), ("i", 1, 0, 0), ("c", 1.5, 0, 0), ("c", 1.5, -3, 0), ("c", 1.5, -3, -6), ("x", 1, 0, 0)]
    assert doc.breaks == [200, 0, 250, None, None, 1500, 500]
    plan = [200, 0, 250, PAUSE, PAUSE, 1500, 500]
    b = batcher_for_model(m, chunk_size=8)
    codes = _record_codes(b)
    try:
        t = b.submit(ssml_request(m, DOC, VOICES), split=True, pause_ms=PAUSE, seed=4321, **GEN)
        chunks = list(t)
        rows = sorted(codes)
        posts = [b.submit(ssml_request(m, DOC, VOICES), split=True, pause_ms=PAUSE, seed=4321, **o, **GEN).audio()
                 for o in POST]
        before = set(codes)
        solo = []
        for k, s in enumerate(doc.spans):
            solo.append(b.submit(voice_request(m, VOICES[s.voice], s.text, s.language),
                                 uniforms=take_uniforms(segment_seed(4321, k), GEN["max_new_tokens"], "cuda"),
                                 **GEN).audio())
        solos = sorted(set(codes) - before)
    finally:
        b.close()
    assert len(rows) == len(solos) == 6
    for r, s in zip(rows, solos):
        assert torch.equal(torch.cat(codes[r]), torch.cat(codes[s]))
    assert [c[2]["segment"] for c in chunks] == sorted(c[2]["segment"] for c in chunks)
    assert all(c[2]["n_segments"] == 6 for c in chunks) and chunks[-1][2]["is_final"]
    audio = np.concatenate([c[0] for c in chunks])
    shaped = [x if (s.speed, s.pitch, s.gain_db) == (1, 0, 0) else _stages(x, s.speed, s.pitch, s.gain_db)
              for x, s in zip(solo, doc.spans)]
    want = join_pauses(shaped, plan)
    assert audio.dtype == np.float32 and np.array_equal(audio, want)
    for g, o in zip(posts, POST):
        enc = "s16" if o["encoding"] == "flac" else o["encoding"]
        twin = _stages(want, o["speed"], 0, 0, o["sample_rate"], enc)
        if o["encoding"] == "flac":
            samples, rate = F.decode(bytes(g))[:2]
            assert rate == o["sample_rate"]
            assert np.array_equal(np.asarray(samples, dtype=np.int16), twin), o
        else:
            assert np.array_equal(g, twin), o


TEXT = "The first sentence is here, and it runs on. A second one follows it here. Third and last sentence now."


def test_plain_document_equals_split_text():
    """<speak>T</speak> is the request split=True makes of T: the same rows, codes and PCM"""
    from faster_qwen3_tts.serving import batcher_for_model, custom_voice_request, ssml_request
    m = _model()
    m.streaming_codec = "stateful"
    voices = {"c": {"speaker": "ryan"}}
    b = batcher_for_model(m, chunk_size=8)
    codes = _record_codes(b)
    try:
        a = b.submit(custom_voice_request(m, TEXT, "ryan", "English", split=True, max_segment_chars=60), split=True,
                     pause_ms=30, seed=99, **GEN).audio()
        first = sorted(codes)
        s = b.submit(ssml_request(m, f"<speak>{TEXT}</speak>", voices, "c", "English", max_segment_chars=60),
                     split=True, pause_ms=30, seed=99, **GEN).audio()
        second = sorted(set(codes) - set(first))
    finally:
        b.close()
    assert len(first) == len(second) == 3
    for r, q in zip(first, second):
        assert torch.equal(torch.cat(codes[r]), torch.cat(codes[q]))
    assert len(a) > 0 and np.array_equal(a, s)


def test_speak_ssml_equals_its_stream():
    m = _model()
    m.streaming_codec = "stateful"
    shot, sr = m.speak_ssml(DOC, VOICES, pause_ms=20, seed=5, pitch=2, **GEN)
    chunks = list(m.speak_ssml_streaming(DOC, VOICES, pause_ms=20, seed=5, pitch=2, **GEN))
    assert sr == 24000 and len(shot[0]) > 0
    assert np.array_equal(shot[0], np.concatenate([c[0] for c in chunks]))
    assert chunks[-1][2]["n_segments"] == 6 and chunks[-1][2]["is_final"]
