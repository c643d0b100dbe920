"""CPU tests of the log-probability plumbing: the host assembly of the kernels' rows (the shifted column 0 and the EOS
term), the float64 reference of oracle/logprob_oracle.py against torch.log_softmax, and the argument checks of the
``*_takes`` calls (fakes, no engine)."""
import inspect
import math
import types

import pytest
import torch

from faster_qwen3_tts import FasterQwen3TTS
from faster_qwen3_tts.logprobs import FrameLogprobs, score
from oracle import logprob_oracle as LO

EOS = 7


def _raw(T, seed):
    g = torch.Generator().manual_seed(seed)
    return -torch.rand(T, 16, generator=g)


def test_column0_is_shifted_across_chunks():
    raw = _raw(10, 0)
    a = FrameLogprobs(-0.25)
    parts = [a.push(raw[:4]), a.push(raw[4:4]), a.push(raw[4:9]), a.push(raw[9:])]
    got = torch.cat(parts)
    assert torch.equal(got, a.frames())
    assert got[0, 0] == -0.25
    assert torch.equal(got[1:, 0], raw[:-1, 0])
    assert torch.equal(got[:, 1:], raw[:, 1:])
    # the value left after the last frame is the EOS term only when the last draw was EOS
    assert a.eos_logprob(EOS, EOS) == float(raw[-1, 0])
    assert a.eos_logprob(3, EOS) is None


def test_chunking_does_not_change_the_assembly():
    raw = _raw(13, 1)
    whole = FrameLogprobs(-1.0)
    whole.push(raw)
    split = FrameLogprobs(-1.0)
    for i in range(13):
        split.push(raw[i:i + 1])
    assert torch.equal(whole.frames(), split.frames())


def test_first_token_eos_and_score():
    a = FrameLogprobs(-0.5)            # the first cb0 was EOS: no frame, the first-token value is the EOS term
    assert a.frames().shape == (0, 16)
    assert a.eos_logprob(EOS, EOS) == -0.5
    s = score(a.frames(), a.eos_logprob(EOS, EOS))
    assert s["frames"] == 0 and s["total_logprob"] == -0.5
    raw = _raw(5, 2)
    b = FrameLogprobs(-0.1)
    rows = b.push(raw)
    s = score(rows, None)
    assert s["eos_logprob"] is None and math.isclose(s["total_logprob"], float(rows.double().sum()), rel_tol=0, abs_tol=1e-12)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_logprob64_matches_log_softmax(dtype):
    g = torch.Generator().manual_seed(4)
    for _ in range(5):
        row = (torch.randn(3072, generator=g) * 4).to(dtype)
        row[torch.randint(0, 3072, (50,), generator=g)] = float("-inf")
        want = torch.log_softmax(row.double(), dim=-1)
        for tok in torch.randint(0, 3072, (20,), generator=g).tolist():
            if math.isinf(float(row[tok])):
                continue
            assert abs(LO.logprob64(row, tok) - float(want[tok])) < 1e-12


def test_processed_row_greedy_and_filters():
    g = torch.Generator().manual_seed(5)
    lg = torch.randn(256, generator=g)
    mask = torch.zeros(256, dtype=torch.bool)
    mask[200:] = True
    greedy = LO.processed_row(lg, do_sample=False, temperature=0.5, top_k=3, top_p=0.5, suppress_mask=mask)
    assert torch.isinf(greedy[200:]).all() and torch.equal(greedy[:200], lg[:200])   # no temperature, no filters
    k1 = LO.processed_row(lg, do_sample=True, temperature=0.9, top_k=1, top_p=1.0)
    tok = int(torch.argmax(lg))
    assert torch.isfinite(k1).sum() == 1 and LO.logprob64(k1, tok) == 0.0
    topp = LO.processed_row(lg, do_sample=True, temperature=0.9, top_k=0, top_p=0.3)
    kept = torch.isfinite(topp)
    assert 1 <= int(kept.sum()) < 256 and bool(kept[tok])


def _fake(max_batch, kind=None):
    base = types.SimpleNamespace(model=types.SimpleNamespace(tts_model_type=kind))
    tg = types.SimpleNamespace(engine=types.SimpleNamespace(max_batch=max_batch))
    return FasterQwen3TTS(base, object(), tg, device="cpu")


def test_takes_argument_checks():
    m = _fake(4, "custom_voice")
    for n in (0, 5, -1):
        with pytest.raises(ValueError, match=f"n_takes={n}"):
            m.generate_custom_voice_takes("hi", "ryan", "English", n_takes=n)
    with pytest.raises(ValueError, match="3 seeds for 2 takes"):
        m.generate_custom_voice_takes("hi", "ryan", "English", n_takes=2, seeds=[1, 2, 3])
    with pytest.raises(ValueError, match="max_batch >= 2"):
        _fake(1).generate_voice_clone_takes("hi", "English", n_takes=1)
    with pytest.raises(ValueError, match="max_batch >= 2"):
        _fake(1, "voice_design").generate_voice_design_takes("hi", "calm", "English")
    assert m._check_takes(3, [5, 6, 7]) == [5, 6, 7]
    assert len(set(m._check_takes(4, None))) == 4


def test_takes_signatures():
    for name in ("generate_voice_clone_takes", "generate_custom_voice_takes", "generate_voice_design_takes"):
        d = {k: v.default for k, v in inspect.signature(getattr(FasterQwen3TTS, name)).parameters.items()}
        assert list(d)[-2:] == ["n_takes", "seeds"] and d["n_takes"] == 4 and d["seeds"] is None
