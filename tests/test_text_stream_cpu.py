"""Incremental text input on the host (no GPU): the commit rule that turns text pieces into token ids, the refusals of
the text-fed entry points, the C ABI of fq3_set_text_rows, and the scheduler's ready-slot selection and cancel."""
import ctypes
import os
import random
import types

import pytest
import torch

from oracle import prompt_cases  # noqa: F401  (puts the package on sys.path)
from faster_qwen3_tts import FasterQwen3TTS
from faster_qwen3_tts.synthetic_frontend import SyntheticOuter
from faster_qwen3_tts.text_stream import PRETOKENIZE_REGEX, TextCommitter, TextFeed, stable_prefix

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TEXTS = [
    "Hello, world! It's 3:45 pm -- we're   late; don't worry.\nNew line here...\n\n  Indented (really) 12345 items.",
    "The quick brown fox jumps over the lazy dog 42 times, isn't it? Yes!!  Absolutely.\t\tTabs too",
    "今天天气很好我们去公园散步吧。然后去吃饭，好不好？",
    "Mixed 中文和English混合 text, with numbers 2024年10月 and emoji-free punctuation: «quotes» — dashes.",
    "supercalifragilisticexpialidocious antidisestablishmentarianism 1234567890 x\n",
]


def _synthetic_tokenizer():
    inner = types.SimpleNamespace(talker=types.SimpleNamespace(
        get_text_embeddings=lambda: types.SimpleNamespace(num_embeddings=4096), device="cpu"))
    return SyntheticOuter(inner)


class _BPETokenizer:
    """A byte-level BPE on the Qwen2 pre-tokenization regex, trained in memory on a toy corpus, behind the two calls
    the text feed makes (``_build_assistant_text`` / ``_tokenize_texts``)."""

    def __init__(self):
        from tokenizers import Regex, Tokenizer, decoders, models, pre_tokenizers, trainers
        tok = Tokenizer(models.BPE())
        tok.pre_tokenizer = pre_tokenizers.Sequence([
            pre_tokenizers.Split(Regex(PRETOKENIZE_REGEX), behavior="isolated"),
            pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=False)])
        tok.decoder = decoders.ByteLevel()
        trainer = trainers.BpeTrainer(vocab_size=600, special_tokens=["<|im_start|>", "<|im_end|>"],
                                      initial_alphabet=pre_tokenizers.ByteLevel.alphabet())
        tok.train_from_iterator(TEXTS * 20 + ["assistant\n", "hello there general kenobi, what's up?"], trainer)
        self.tok = tok

    @staticmethod
    def _build_assistant_text(text):
        return f"<|im_start|>assistant\n{text}<|im_end|>\n<|im_start|>assistant\n"

    def _tokenize_texts(self, texts):
        return [torch.tensor([self.tok.encode(t).ids], dtype=torch.long) for t in texts]


def _random_split(text, rng):
    cuts = sorted(rng.sample(range(1, len(text)), k=rng.randint(0, min(len(text) - 1, 25)))) if len(text) > 1 else []
    return [text[a:b] for a, b in zip([0] + cuts, cuts + [len(text)])]


@pytest.mark.parametrize("which", ["synthetic", "bpe"])
def test_commit_rule_never_retracts_and_closes_on_the_one_shot_ids(which):
    tok = _synthetic_tokenizer() if which == "synthetic" else _BPETokenizer()
    if which == "bpe":   # the body of the template is the text's own tokens
        ids = tok._tokenize_texts([tok._build_assistant_text("Hello there")])[0][0].tolist()
        assert len(ids) > 8
    rng = random.Random(1234)
    runs = 0
    for text in TEXTS:
        want = tok._tokenize_texts([tok._build_assistant_text(text)])[0][0].tolist()[3:-5]
        for _ in range(60):
            c = TextCommitter(tok)
            seen = []
            for piece in _random_split(text, rng):
                c.push(piece)
                assert c.ids[: len(seen)] == seen, "committed ids were retracted"
                seen = list(c.ids)
                assert seen == want[: len(seen)]
            c.close()
            assert c.ids == want
            runs += 1
    assert runs == 300


def test_commit_rule_holds_back_the_last_pre_token():
    assert stable_prefix("hello wor") == "hello"
    assert stable_prefix("it'") == "it"
    assert stable_prefix("a  ") == "a"
    assert stable_prefix("12") == "1"
    assert stable_prefix("") == ""
    c = TextCommitter(_synthetic_tokenizer())
    c.push("hello wor")
    assert len(c.ids) == 1       # "hello" committed, "wor" may still grow
    c.push("ld")
    assert len(c.ids) == 1
    c.push(" ")
    assert len(c.ids) == 2
    c.close()
    with pytest.raises(RuntimeError):
        c.push("more")


def _feed_model():
    tok = _synthetic_tokenizer()
    talker = types.SimpleNamespace(device="cpu")
    return types.SimpleNamespace(model=types.SimpleNamespace(
        model=types.SimpleNamespace(talker=talker), _build_assistant_text=tok._build_assistant_text,
        _tokenize_texts=tok._tokenize_texts))


def test_empty_text_is_refused():
    for pieces in ([], [""], ["   "]):
        f = TextFeed(_feed_model(), max_rows=8)
        for p in pieces:
            f.push(p)
        with pytest.raises(ValueError, match="without any text"):
            f.close()


def _public_model():
    base = types.SimpleNamespace(model=types.SimpleNamespace(tts_model_type="custom_voice"),
                                 _build_assistant_text=SyntheticOuter._build_assistant_text)
    return FasterQwen3TTS(base, object(), object(), device="cpu")


def test_text_streaming_refuses_non_streaming_layout_and_icl():
    m = _public_model()
    with pytest.raises(ValueError, match="non_streaming_mode"):
        next(m.generate_custom_voice_text_streaming(iter(["hi"]), "aiden", "English", non_streaming_mode=True))
    m.model.model.tts_model_type = "voice_design"
    with pytest.raises(ValueError, match="non_streaming_mode"):
        next(m.generate_voice_design_text_streaming(iter(["hi"]), "calm", "English", non_streaming_mode=True))
    m.model.model.tts_model_type = "base"
    with pytest.raises(ValueError, match="ICL"):
        next(m.generate_voice_clone_text_streaming(iter(["hi"]), "English", ref_audio="ref.wav", ref_text="words",
                                                   xvec_only=False))
    vcp = dict(ref_spk_embedding=[torch.zeros(4)], ref_code=[torch.zeros(3, 16, dtype=torch.long)],
               x_vector_only_mode=[False], icl_mode=[True])
    m = FasterQwen3TTS(_synthetic_tokenizer(), object(), object(), device="cpu")   # resolving ICL reads ref_text ids
    with pytest.raises(ValueError, match="ICL"):
        next(m.generate_voice_clone_text_streaming(iter(["hi"]), "English", voice_clone_prompt=vcp, ref_text="words"))


def test_set_text_rows_c_abi():
    from faster_qwen3_tts.engine import EXPORTS, LIB_PATH, build_extension, load_library
    build_extension()
    assert "fq3_set_text_rows" in EXPORTS
    lib = load_library()
    assert [t for t in lib.fq3_set_text_rows.argtypes] == [ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32]
    assert lib.fq3_set_text_rows(None, 0, 1, 1) == -1          # FQ3_ERR_INVALID: null engine
    assert b"null" in lib.fq3_last_error()
    hdr = open(os.path.join(ROOT, "include", "fq3_engine.h")).read()
    assert "int fq3_set_text_rows(fq3_engine* e, int32_t slot, int32_t trailing_len, int32_t open);" in hdr
    assert os.path.exists(LIB_PATH)


# ---- BatchScheduler against a fake engine ----------------------------------------------------------------------
class _FakeFeed:
    def __init__(self, n_rows=0, closed=False):
        self.n_rows, self.closed = n_rows, closed

    def update(self):
        return self.n_rows


class _FakeEngine:
    """Slots emit frames like the kernels do: an open slot runs only while row gen_step exists."""

    def __init__(self, max_batch):
        self.max_batch = max_batch
        self.gen_step0, self.rows, self.launches = {}, {}, []
        self.step = {}

    def set_text_rows(self, slot, n, open):
        assert n >= self.rows.get(slot, (0, True))[0], "rows shrank"
        self.rows[slot] = (n, open)

    def _run(self, slot, n_frames):
        n, open = self.rows.get(slot, (10 ** 6, False))
        k = n_frames if not open else max(0, min(n_frames, n - self.gen_step0[slot] - self.step[slot]))
        self.step[slot] += k
        return k

    def decode_chunk(self, n_frames, slot=0):
        self.launches.append([slot])
        k = self._run(slot, n_frames)
        return torch.zeros(k, 16, dtype=torch.long), types.SimpleNamespace(frames_emitted=k, finished=0)

    def decode_chunk_batch(self, slots, n_frames):
        self.launches.append(list(slots))
        res = [types.SimpleNamespace(frames_emitted=self._run(s, n_frames), finished=0) for s in slots]
        return torch.zeros(len(slots), n_frames, 16, dtype=torch.long), res


def test_batch_scheduler_launches_ready_slots_only_and_cancel_frees(monkeypatch):
    from faster_qwen3_tts import batching

    def fake_begin(engine, *a, slot=None, trailing_len=None, **kw):
        engine.gen_step0[slot] = 0
        engine.step[slot] = 0
        engine.rows.pop(slot, None)

    monkeypatch.setattr(batching, "begin_fused", fake_begin)
    eng = _FakeEngine(3)
    sched = batching.BatchScheduler(eng, None, None, None, None)
    z = torch.zeros(1)
    plain = sched.submit(z, z, z, z, tag="plain")
    fa, fb = _FakeFeed(0), _FakeFeed(5)
    a = sched.submit(z, z, z, z, tag="a", feed=fa)
    b = sched.submit(z, z, z, z, tag="b", feed=fb)
    assert not sched.has_capacity()
    assert not a.ready() and b.ready() and plain.ready()
    out = sched.step(4)
    assert eng.launches[-1] == [plain.slot, b.slot]           # the starved slot is not launched
    assert {rq.tag: int(c.shape[0]) for rq, c in out} == {"plain": 4, "b": 4}
    out = sched.step(4)
    assert {rq.tag: int(c.shape[0]) for rq, c in out} == {"plain": 4, "b": 1}   # b stops at its last row
    assert not b.ready()
    fb.closed = True                                          # closed text: ready again, runs on tts_pad
    fa.n_rows = 2
    sched.step(4)
    assert eng.launches[-1] == [plain.slot, a.slot, b.slot]
    assert eng.rows[b.slot] == (5, False) and eng.rows[a.slot] == (2, True)
    assert a.frames == 2 and not a.ready()
    sched.cancel(a)
    assert sched.has_capacity() and a.slot not in sched.active
    sched.cancel(a)                                           # idempotent
    assert sched.free.count(a.slot) == 1
    c = sched.submit(z, z, z, z, tag="c")
    assert c.slot == a.slot
    sched.cancel(plain)
    sched.cancel(b)
    sched.cancel(c)
    assert sched.step(4) == [] and len(sched) == 0


def test_voice_clone_text_streaming_takes_list_form_prompts():
    """A list of prompt items (what upstream ``create_voice_clone_prompt`` returns) is resolved like the other clone
    entry points resolve it: x-vector items pass validation (and then need the engine), ICL items are refused."""
    tok = _synthetic_tokenizer()
    m = FasterQwen3TTS(tok, object(), object(), device="cpu")
    xvec = [types.SimpleNamespace(ref_code=None, ref_spk_embedding=torch.zeros(4), x_vector_only_mode=True,
                                  icl_mode=False, ref_text=None)]
    with pytest.raises(RuntimeError, match="fq3 engine"):
        next(m.generate_voice_clone_text_streaming(iter(["hi"]), "English", voice_clone_prompt=xvec))
    icl = [types.SimpleNamespace(ref_code=torch.zeros(3, 16, dtype=torch.long), ref_spk_embedding=torch.zeros(4),
                                 x_vector_only_mode=False, icl_mode=True, ref_text="the reference words")]
    with pytest.raises(ValueError, match="ICL"):
        next(m.generate_voice_clone_text_streaming(iter(["hi"]), "English", voice_clone_prompt=icl))


def test_ready_needs_rows_ahead_and_ends_at_max_new_tokens():
    from faster_qwen3_tts.batching import SlotRequest
    f = _FakeFeed(7)
    rq = SlotRequest(slot=0, tag=0, max_new_tokens=10, feed=f, rows_ahead=8)
    assert not rq.ready()                 # a full chunk of rows (8) does not exist yet
    f.n_rows = 8
    assert rq.ready()
    rq.frames = 8
    f.n_rows = 9
    assert not rq.ready()
    f.n_rows = 10                         # rows up to max_new_tokens suffice: the launch ends the request
    assert rq.ready()
    rq.frames, f.n_rows = 10, 10          # reached max_new_tokens with open text: launched so that it reports finished
    assert rq.ready()
