"""The single-request drivers on a fake K3 engine, without a GPU: ``begin_fused``, ``fast_generate``,
``fast_generate_streaming`` and ``generate_text_streaming`` make the engine calls of one request on the slot the graph
handles drive (here 3), with the launch sizes, returned codes, timing keys and shifted log-probabilities they document,
and draw their default uniforms from the global generator once per request."""
import types

import pytest
import torch

from oracle import prompt_cases  # noqa: F401  (puts the package on sys.path)
from faster_qwen3_tts import text_stream
from faster_qwen3_tts.engine import SamplingParams
from faster_qwen3_tts.generate import begin_fused, fast_generate
from faster_qwen3_tts.streaming import fast_generate_streaming
from faster_qwen3_tts.synthetic_frontend import SyntheticOuter

SLOT, H, V, EOS, FIRST, FIRST_LP = 3, 4, 6, 2, 5, -0.25


def _raw_lp(g):
    """the kernel's log-probability row of frame g (column 0: the cb0 drawn after it)"""
    return [-(g * 16 + k + 1) / 64 for k in range(16)]


class _Engine:
    """A K3 engine whose request emits ``total`` frames and then draws EOS; records every call a driver makes.  A slot
    with open text runs only while its next row exists, as the kernels do."""
    has_prefill, loaded, device, H = True, True, torch.device("cpu"), H
    max_batch, max_slots, max_seq_len, eos = 4, 8, 64, EOS
    time_kernels, last_kernel_ms = False, None

    def __init__(self, total):
        self.total, self.done, self.calls, self.text, self.gen_step0 = total, 0, [], {}, {}
        self.uniforms = None

    def _prefilled(self, x, pad, slot):
        self.calls.append(("prefill", [int(slot)], int(pad)))
        return torch.arange(V, dtype=torch.float32) + float(x.sum()), x.reshape(-1, H)[-1]

    def prefill(self, x, pad, slot=0):
        return self._prefilled(x, pad, slot)

    def prefill_batch(self, rows, pads, slots):
        assert len(rows) == len(pads) == len(slots) == 1
        lg, hid = self._prefilled(rows[0], pads[0], slots[0])
        return lg[None], hid[None]

    def sample_logits(self, logits, sp, u=0.0, suppress_special=False, eos_id=-1, suppress_eos=False,
                      return_logprob=False):
        self.calls.append(("sample_logits", sp, u, suppress_special, eos_id, suppress_eos, return_logprob))
        tok = torch.tensor([FIRST if self.total else EOS])
        return (tok, torch.tensor([FIRST_LP])) if return_logprob else tok

    def set_generation_state(self, n_left_pad, rope_delta, slot=0):
        self.calls.append(("set_generation_state", n_left_pad, rope_delta, slot))

    def begin_request(self, *, uniforms, past_hidden, trailing_text, tts_pad, sp_talker, sp_predictor, **kw):
        self.calls.append(("begin_request", tuple(sorted(kw.items())), sp_talker, sp_predictor))
        self.uniforms = uniforms
        self.gen_step0[kw["slot"]] = kw["gen_step"]

    def set_text_rows(self, slot, n, open):
        self.text[slot] = (int(n), bool(open))

    def decode_chunk(self, n_frames, out=None, slot=0, logprobs=None):
        self.calls.append(("decode_chunk", n_frames, slot, bool(logprobs), self.text.get(slot)))
        k = min(n_frames, self.total - self.done)
        if self.text.get(slot, (0, False))[1]:
            k = min(k, self.text[slot][0] - self.done)
        g = range(self.done, self.done + k)
        self.done += k
        codes = torch.tensor([[100 * i + c for c in range(16)] for i in g], dtype=torch.long).reshape(k, 16)
        fin = self.done >= self.total
        res = types.SimpleNamespace(frames_emitted=k, finished=int(fin), next_token=EOS if fin else FIRST)
        if logprobs:
            return codes, torch.tensor([_raw_lp(i) for i in g], dtype=torch.float32).reshape(k, 16), res
        return codes, res

    def decode_chunk_batch(self, *a, **kw):
        raise AssertionError("a single request is launched with the single-sequence kernel")


def _handles(eng, do_sample):
    pg = types.SimpleNamespace(engine=eng, do_sample=do_sample, sampling=lambda: SamplingParams(do_sample, 7, 0.8, 0.9))
    tg = types.SimpleNamespace(engine=eng, slot=SLOT)
    return pg, tg


def _prompt(P=5, pad=2):
    g = torch.Generator().manual_seed(P)
    tam = torch.ones(1, P, dtype=torch.long)
    tam[0, :pad] = 0
    return torch.randn(1, P, H, generator=g), tam, torch.randn(1, 3, H, generator=g), torch.zeros(1, 1, H)


CFG = types.SimpleNamespace(codec_eos_token_id=EOS)
GEN = dict(max_new_tokens=8, min_new_tokens=2, temperature=0.7, top_k=30, top_p=0.95, repetition_penalty=1.1)


def _latch_calls(tie, pad, do_sample, u0, logprob, trailing_len=None, first=FIRST):
    sp = SamplingParams(do_sample, GEN["top_k"], GEN["temperature"], GEN["top_p"], 1.0)
    sp_t = SamplingParams(do_sample, GEN["top_k"], GEN["temperature"], GEN["top_p"], GEN["repetition_penalty"])
    begin = dict(first_token=first, gen_step=0, max_new_tokens=GEN["max_new_tokens"],
                 min_new_tokens=GEN["min_new_tokens"], n_left_pad=pad, prefill_len=int(tie.shape[1]), rope_delta=-pad,
                 slot=SLOT, trailing_len=trailing_len)
    return [("prefill", [SLOT], pad), ("sample_logits", sp, u0, True, EOS, True, logprob),
            ("set_generation_state", pad, -pad, SLOT),
            ("begin_request", tuple(sorted(begin.items())), sp_t, SamplingParams(do_sample, 7, 0.8, 0.9))]


@pytest.mark.parametrize("logprob", [False, True])
@pytest.mark.parametrize("uniforms", ["default", "given", "greedy"])
def test_begin_fused_latches_one_row_on_the_graph_slot(logprob, uniforms):
    eng = _Engine(5)
    do_sample = uniforms != "greedy"
    pg, tg = _handles(eng, do_sample)
    tie, tam, tth, tpe = _prompt()
    torch.manual_seed(11)
    want_u = torch.rand(GEN["max_new_tokens"] + 1, 16) if do_sample else None   # the request's draw
    given = want_u.clone() if uniforms == "given" else None
    torch.manual_seed(11)
    got = begin_fused(eng, None, tie, tam, tth, tpe, CFG, pg, tg, do_sample=do_sample, uniforms=given,
                      **({"logprob": True} if logprob else {}), **GEN)
    after = torch.rand(4)
    u0 = float(want_u[0, 0]) if do_sample else 0.0
    assert eng.calls == _latch_calls(tie, 2, do_sample, u0, logprob)
    assert (eng.uniforms is None) if not do_sample else torch.equal(eng.uniforms, want_u)
    torch.manual_seed(11)   # the global generator moved by the request's one draw, and only when none was given
    if uniforms == "default":
        torch.rand(GEN["max_new_tokens"] + 1, 16)
    assert torch.equal(after, torch.rand(4))
    if logprob:
        first, lp = got
        assert int(first) == FIRST and lp == FIRST_LP
    else:
        assert int(got) == FIRST
    assert (tg.prefill_len, tg.n_left_pad, tg.rope_delta) == (5, 2, -2)


def _shifted(frames, first_lp=FIRST_LP):
    rows = torch.tensor([_raw_lp(g) for g in frames], dtype=torch.float32).reshape(-1, 16)
    out = rows.clone()
    if len(frames):
        out[0, 0] = first_lp
        out[1:, 0] = rows[:-1, 0]
    return out


def _codes(frames):
    return torch.tensor([[100 * g + c for c in range(16)] for g in frames], dtype=torch.long)


@pytest.mark.parametrize("return_logprobs", [False, True])
@pytest.mark.parametrize("total", [5, 0])
def test_fast_generate_runs_one_request_in_256_frame_launches(return_logprobs, total):
    eng = _Engine(total)
    pg, tg = _handles(eng, False)
    tie, tam, tth, tpe = _prompt()
    codes, timing = fast_generate(None, tie, tam, tth, tpe, CFG, pg, tg, do_sample=False,
                                  return_logprobs=return_logprobs, **GEN)
    assert eng.calls == _latch_calls(tie, 2, False, 0.0, return_logprobs, first=FIRST if total else EOS) + \
        [("decode_chunk", 256, SLOT, return_logprobs, None)]
    want = {"prefill_ms", "decode_s", "steps", "ms_per_step", "steps_per_s"}
    if total:
        assert torch.equal(codes, _codes(range(total)))
    else:
        assert codes is None
    assert timing["steps"] == total
    if return_logprobs:
        want |= {"logprobs", "eos_logprob"}
        assert torch.equal(timing["logprobs"], _shifted(range(total)))
        assert timing["eos_logprob"] == (_raw_lp(total - 1)[0] if total else FIRST_LP)
    assert set(timing) == want


@pytest.mark.parametrize("return_logprobs", [False, True])
def test_fast_generate_streaming_runs_one_request_in_chunk_size_launches(return_logprobs):
    eng = _Engine(5)
    pg, tg = _handles(eng, False)
    tie, tam, tth, tpe = _prompt()
    chunks = list(fast_generate_streaming(None, tie, tam, tth, tpe, CFG, pg, tg, do_sample=False, chunk_size=2,
                                          return_logprobs=return_logprobs, **GEN))
    assert eng.calls == _latch_calls(tie, 2, False, 0.0, return_logprobs) + \
        [("decode_chunk", 2, SLOT, return_logprobs, None)] * 3
    spans = [range(0, 2), range(2, 4), range(4, 5)]
    assert len(chunks) == 3
    for i, ((codes, tm), span) in enumerate(zip(chunks, spans)):
        assert torch.equal(codes, _codes(span))
        keys = {"chunk_index", "chunk_steps", "prefill_ms", "decode_ms", "total_steps_so_far", "is_final"}
        assert (tm["chunk_index"], tm["chunk_steps"], tm["total_steps_so_far"], tm["is_final"]) == \
            (i, len(span), span.stop, i == 2)
        assert i == 0 or tm["prefill_ms"] == 0
        if return_logprobs:
            keys |= {"logprobs"} | ({"eos_logprob"} if i == 2 else set())
            assert torch.equal(tm["logprobs"], _shifted(range(5))[span.start:span.stop])
        assert set(tm) == keys
    if return_logprobs:
        assert chunks[-1][1]["eos_logprob"] == _raw_lp(4)[0]


def _text_model(eng, do_sample):
    emb = torch.nn.Embedding(4096, H)
    talker = types.SimpleNamespace(device="cpu", get_text_embeddings=lambda: emb, text_projection=lambda x: x)
    tok = SyntheticOuter(types.SimpleNamespace(talker=talker))
    tok.model.speech_tokenizer, tok.model.config = None, types.SimpleNamespace(talker_config=CFG)
    pg, tg = _handles(eng, do_sample)
    return types.SimpleNamespace(model=tok, predictor_graph=pg, talker_graph=tg, sample_rate=24000)


def test_generate_text_streaming_runs_one_request_on_the_graph_slot(monkeypatch):
    eng = _Engine(7)
    model = _text_model(eng, False)
    tie, tam, _, tpe = _prompt()

    def prompt(model, feed, **kw):
        feed.start(torch.zeros(H), torch.float32)
        return tie, tam, tpe
    monkeypatch.setattr(text_stream, "build_prompt", prompt)
    pieces = ["one two three ", "four five six seven ", "eight.", "never read"]
    got = list(text_stream.generate_text_streaming(model, iter(pieces), language="English", chunk_size=2,
                                                   do_sample=False, to_host=False, **GEN))
    rows = [(2, True), (6, True), (6, True), (7, True)]   # announced before each launch: one frame of rows ahead
    assert eng.calls == _latch_calls(tie, 2, False, 0.0, False, trailing_len=0) + \
        [("decode_chunk", 2, SLOT, False, r) for r in rows]
    spans = [range(0, 2), range(2, 4), range(4, 6), range(6, 7)]
    assert len(got) == 4
    for i, ((codes, sr, tm), span) in enumerate(zip(got, spans)):
        assert sr == 24000 and torch.equal(codes, _codes(span))
        assert set(tm) == {"chunk_index", "chunk_steps", "prefill_ms", "decode_ms", "total_steps_so_far", "is_final",
                           "text_wait_ms"}
        assert (tm["chunk_index"], tm["chunk_steps"], tm["total_steps_so_far"], tm["is_final"]) == \
            (i, len(span), span.stop, i == 3)
        assert i == 0 or tm["prefill_ms"] == 0
        assert tm["decode_ms"] >= 0 and tm["text_wait_ms"] >= 0
