"""GPU tests of the ``*_takes`` calls: n takes of one request in one batched prefill and one batched decode.

Take i must be exactly the same request run alone with take i's uniforms (``take_uniforms(seeds[i])``): codes
bit-identical, PCM bit-identical to its one-shot decode and, with the stateful codec, to the request streamed alone;
takes of equal length share one codec call; its score must be the sum of its returned log-probabilities; the refusals raise
before anything is launched."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

TEXT = "Several takes of the same sentence, rendered side by side."


def _model(max_batch=4):
    from faster_qwen3_tts import FasterQwen3TTS
    return FasterQwen3TTS.from_synthetic("tiny", dtype=torch.bfloat16, max_seq_len=256, seed=8, max_batch=max_batch)


def _alone(m, prep, ref_codes, seed, gen):
    """what generate_voice_clone / generate_custom_voice do, with take `seed`'s uniforms"""
    from faster_qwen3_tts.generate import fast_generate
    from faster_qwen3_tts.model import take_uniforms
    mm, talker, config, tie, tam, tth, tpe = prep
    talker.rope_deltas = None
    codes, timing = fast_generate(talker=talker, talker_input_embeds=tie, attention_mask=tam, trailing_text_hiddens=tth,
                                  tts_pad_embed=tpe, config=config, predictor_graph=m.predictor_graph,
                                  talker_graph=m.talker_graph, uniforms=take_uniforms(seed, gen["max_new_tokens"]),
                                  return_logprobs=True, **gen)
    audio, _ = m._decode_all(mm.speech_tokenizer, codes, ref_codes)
    return codes.cpu(), audio[0], timing


def _streamed(m, prep, ref_codes, seed, gen):
    """the same request streamed alone (stateful codec: its PCM is the one-shot decode of its codes)"""
    from faster_qwen3_tts.model import take_uniforms
    _, talker, _, tie, tam, tth, tpe = prep
    talker.rope_deltas = None
    parts = [a for a, _, _ in m.stream_from_embeds(tie, tam, tth, tpe, ref_codes=ref_codes, chunk_size=8,
                                                    uniforms=take_uniforms(seed, gen["max_new_tokens"]), **gen)]
    return np.concatenate(parts)


@pytest.mark.parametrize("kind,codec_mode,fixed_len", [("custom_voice", "window", False),
                                                       ("voice_clone_icl", "window", True),
                                                       ("custom_voice", "stateful", True),
                                                       ("voice_clone_icl", "stateful", False)])
def test_each_take_equals_the_request_run_alone(kind, codec_mode, fixed_len, monkeypatch):
    # the ICL prompt crosses 192 cached keys while generating: from there a lone request's single-sequence kernel would
    # switch to its split-key attention, which the batched kernel does not have (as in test_gpu_serving.py)
    monkeypatch.setenv("FQ3_ATTN_SPLIT", "0")
    m = _model()
    m.streaming_codec = codec_mode
    gen = dict(max_new_tokens=40, min_new_tokens=40 if fixed_len else 2, temperature=0.9, top_k=50, top_p=1.0,
               do_sample=True, repetition_penalty=1.05)
    seeds = [11, 12, 13, 14]
    st = m.model.model.speech_tokenizer
    batches = []
    decode = st.decode
    monkeypatch.setattr(st, "decode", lambda d: (batches.append(int(d["audio_codes"].shape[0])), decode(d))[1])
    if kind == "custom_voice":
        spk = "ryan"
        audios, sr, scores = m.generate_custom_voice_takes(TEXT, spk, "English", n_takes=4, seeds=seeds, **gen)
        with torch.inference_mode():
            prep = m._prepare_generation_custom(TEXT, "English", spk)
        ref_codes = None
    else:
        audios, sr, scores = m.generate_voice_clone_takes(TEXT, "English", ref_audio="ref.wav", ref_text="ref words",
                                                          n_takes=4, seeds=seeds, **gen)
        with torch.inference_mode():
            *prep, ref_codes = m._prepare_generation(text=TEXT, language="English", ref_audio="ref.wav",
                                                     ref_text="ref words", non_streaming_mode=False)
        assert ref_codes is not None
    lengths = [s["frames"] for s in scores]
    assert sorted(batches, reverse=True) == sorted([lengths.count(T) for T in set(lengths)], reverse=True)
    if fixed_len:   # all takes have one length: their PCM comes from ONE codec call of 4 rows
        assert batches == [4]
    assert sr == m.sample_rate and len(audios) == len(scores) == 4
    for i, s in enumerate(seeds):
        with torch.inference_mode():
            codes, audio, timing = _alone(m, tuple(prep), ref_codes, s, gen)
        sc = scores[i]
        assert sc["seed"] == s and sc["frames"] == codes.shape[0]
        assert torch.equal(sc["logprobs"], timing["logprobs"])
        assert sc["eos_logprob"] == timing["eos_logprob"]
        want_total = float(sc["logprobs"].double().sum()) + (sc["eos_logprob"] or 0.0)
        assert abs(sc["total_logprob"] - want_total) < 1e-9
        assert (sc["logprobs"] <= 0).all()
        assert audios[i].shape == audio.shape and np.array_equal(audios[i], audio), i
        if codec_mode == "stateful":
            with torch.inference_mode():
                streamed = _streamed(m, tuple(prep), ref_codes, s, gen)
            assert streamed.shape == audio.shape and np.array_equal(streamed, audios[i]), i
    assert len({float(s["total_logprob"]) for s in scores}) > 1   # the takes differ


def test_takes_refusals_before_launch():
    m = _model(max_batch=4)
    n0 = m.engine.launch_count
    with pytest.raises(ValueError, match="n_takes=5"):
        m.generate_custom_voice_takes(TEXT, "ryan", "English", n_takes=5)
    with pytest.raises(ValueError, match="n_takes=0"):
        m.generate_voice_design_takes(TEXT, "calm", "English", n_takes=0)
    with pytest.raises(ValueError, match="seeds"):
        m.generate_voice_clone_takes(TEXT, "English", ref_audio="ref.wav", ref_text="ref words", n_takes=2, seeds=[1])
    assert m.engine.launch_count == n0
    one = _model(max_batch=1)
    n1 = one.engine.launch_count
    with pytest.raises(ValueError, match="max_batch >= 2"):
        one.generate_custom_voice_takes(TEXT, "ryan", "English", n_takes=1)
    assert one.engine.launch_count == n1
