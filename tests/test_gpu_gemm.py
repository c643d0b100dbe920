"""The dense-layer GEMM of the prefill and the codec (fq3gemm::gemm, through the fq3_debug_conv_gemm probe) against the
float64 reference of tests/util_gemm.py, at the shapes and epilogues where an implicit-GEMM kernel goes wrong: BK = 32
and 64 with one and several k-chunks, N tails inside a 32-column group and inside a 96-column tile, M tails, causal
shifts longer than the sequence, batches of sequences with different data, history rows, both ring depths (KIND 0 / 1),
and every epilogue.

Two bars per output:
  * elementwise, |kernel - reference| <= the bound util_gemm derives (fp32 accumulation error carried through the
    epilogue, one bf16 ulp per rounding point, __sinf's error for SnakeBeta);
  * an exact-match fraction.  An output differs from the correctly rounded reference only where the fp64 value lies
    within the accumulation error of a bf16 rounding boundary: about sqrt(K) 2^-24 / 2^-8, 5e-4 at K = 1024.  So >= 99 %
    of Yraw outputs (mode 1's included) must equal the reference bit for bit.  This is what catches a dropped, added or
    misplaced rounding point: it moves an output by about one ulp, inside the elementwise bar.  Measured on an H100
    (sm_90a): >= 99.87 % at K <= 1024, and 99.44 % at K = 7 x 1024, four times the sqrt(K) estimate there: the wgmma
    accumulator's error grows like K / 16 roundings that do not cancel (truncation), which the elementwise bound
    already assumes.  Yact adds __sinf: with the tested |ib| <= 1.6 and |z| = |ea x| up to ~150, its error
    2 ib (2^-21.41 + |z| 2^-22) is at most ~1e-4, and flips a rounding with probability 2 err / ulp(y); averaged over the
    outputs that is a few 0.1 % (the test prints the estimate), so >= 98.5 % of Yact outputs must be exact.
Bit-exact invariants need no reference: a batch row equals its single-sequence run (KIND 0 against KIND 1), rows
[0, T1) do not depend on later rows, the first N1 columns do not depend on later weight rows, and history rows reproduce
the one-shot tail."""
import math

import pytest
import torch

from util_gemm import conv_acc, epilogue, sin_err, ulp

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from faster_qwen3_tts.engine import EngineError, debug_conv_gemm

RAW_EXACT = 0.99
ACT_EXACT = 0.985
WORST = {}


def _inputs(B, rows, Cin, N, taps, seed, x_std=1.0):
    g = torch.Generator().manual_seed(seed)
    X = (torch.randn(B, rows, Cin, generator=g) * x_std).to(torch.bfloat16).cuda()
    W = (torch.randn(N, taps, Cin, generator=g) / math.sqrt(taps * Cin)).to(torch.bfloat16).cuda()
    return X, W, g


def _params(g, N, epi, B, T):
    """bias / scale / residual / SnakeBeta parameters of an epilogue spec (modular arrays shorter than N on purpose)"""
    p = {}
    if "bias" in epi:
        p["bias"] = (torch.randn(max(8, N // 2), generator=g) * 0.5).cuda()
    if "scale" in epi:
        p["scale"] = (torch.rand(max(8, N // 4), generator=g) + 0.5).cuda()
    if "res" in epi:
        p["R"] = torch.randn(B, T, N, generator=g).to(torch.bfloat16).cuda()
    if "act" in epi:
        m = max(8, N // 2)
        p["ea"] = torch.exp(torch.rand(m, generator=g) * 3.5 - 1.2).cuda()          # exp(alpha): 0.3 .. 10
        p["ib"] = (1.0 / (torch.exp(torch.rand(m, generator=g) * 1.5 - 0.5) + 1e-9)).cuda()   # 0.37 .. 1.6
    return p


def _check(label, got, ref, bar, min_exact):
    assert torch.isfinite(got).all(), label
    g = got.double()
    err = (g - ref).abs()
    ratio = float((err / bar).max())
    exact = float((g == ref).double().mean())
    w = WORST.setdefault(label.split()[0], [0.0, 1.0])
    w[0], w[1] = max(w[0], ratio), min(w[1], exact)
    print(f"{label}: worst error / bar {ratio:.3f}, exact {exact:.5f}")
    assert ratio <= 1.0, (label, ratio, float(err.max()))
    assert exact >= min_exact, (label, exact)


def _act_flip_estimate(ref, p, N):
    """expected fraction of Yact outputs __sinf's error can move across a rounding boundary"""
    cols = torch.arange(N, device=ref["raw"].device)
    a = p["ea"].double()[cols % p["ea"].numel()]
    b = p["ib"].double()[cols % p["ib"].numel()]
    e = 2.0 * b * sin_err(a * ref["raw"])
    return float(torch.clamp(2.0 * e / ulp(ref["act"]), max=1.0).mean())


# (Cin, N, T, taps, dil, batch, epilogue); mode 0 unless the epilogue names "swiglu" / "gelu".  "hist" prepends
# (taps-1)*dil + 3 history rows read through x_row0 / x_rows.
CASES = [
    (32, 8, 1, 1, 1, 1, "bias"),                 # BK 32, one k-chunk, N = one 8-column vector, one output row
    (96, 40, 5, 2, 1, 3, "bias scale res"),      # BK 32, three k-chunks, N ends inside the second 32-column group
    (64, 96, 127, 7, 1, 1, "raw act"),           # BK 64, exactly one N tile, T one short of an M tile
    (1024, 104, 128, 1, 1, 1, "res"),            # BK 64, 16 k-chunks, N 8 columns into a second tile, T = one M tile
    (32, 200, 129, 7, 3, 3, "act"),              # Yact only, T one into a second M tile, three sequences
    (96, 1544, 300, 7, 9, 1, "bias raw act"),    # shift 54, N tail of 8 in the 17th tile
    (64, 40, 5, 7, 9, 3, "bias"),                # shift 54 > T: six of seven taps read only padding
    (1024, 1544, 300, 1, 1, 1, "bias scale res"),
    (64, 1544, 300, 7, 3, 5, "bias raw act"),    # 255 tiles: KIND 0 with BK 64
    (96, 1544, 129, 2, 1, 5, "scale res"),       # 170 tiles / 255 at T 300 below: KIND 1 and KIND 0 with BK 32
    (96, 1544, 300, 2, 1, 5, "bias res"),
    (1024, 8, 300, 7, 3, 3, "bias raw act"),
    (1024, 200, 129, 2, 1, 3, "gelu bias"),      # mode 2
    (32, 104, 300, 7, 3, 1, "gelu bias scale res"),
    (64, 96, 129, 7, 3, 3, "hist bias raw act"),
    (96, 200, 5, 7, 9, 1, "hist res"),           # 57 history rows, 5 new
    (1024, 1600, 300, 1, 1, 1, "swiglu"),        # mode 1: the talker's gate/up shape class, N tail of 64 in a tile
    (64, 160, 129, 1, 1, 3, "swiglu"),
    (32, 32, 1, 1, 1, 1, "swiglu"),
    (96, 160, 128, 2, 1, 1, "swiglu"),
]


def _ids(c):
    return f"Cin{c[0]}-N{c[1]}-T{c[2]}-k{c[3]}d{c[4]}-b{c[5]}-" + c[6].replace(" ", "+")


@pytest.mark.parametrize("case", CASES, ids=[_ids(c) for c in CASES])
def test_gemm_vs_float64_reference(case):
    Cin, N, T, taps, dil, B, epi = case
    mode = 1 if "swiglu" in epi else (2 if "gelu" in epi else 0)
    h = (taps - 1) * dil + 3 if "hist" in epi else 0
    x_std = 4.0 if "act" in epi else 1.0      # SnakeBeta arguments |ea x| up to ~150, far outside [-pi, pi]
    X, W, g = _inputs(B, h + T, Cin, N, taps, seed=CASES.index(case), x_std=x_std)
    p = _params(g, N, epi, B, T)
    want_act = "act" in epi
    want_raw = mode != 0 or "raw" in epi or not want_act
    Yraw, Yact = debug_conv_gemm(X, W, mode=mode, dil=dil, T=T, raw=want_raw, act=want_act, x_row0=h, history=h > 0,
                                 **p)
    acc, mag = conv_acc(X, W, dil, T=T, x_row0=h, history=h > 0)
    ref = epilogue(acc, mag, taps * Cin, mode, bias=p.get("bias"), scale=p.get("scale"), R=p.get("R"), ea=p.get("ea"),
                   ib=p.get("ib"), act=want_act)
    label = ["mode0", "swiglu", "gelu"][mode]
    if Yraw is not None:
        _check(f"{label} Yraw {_ids(case)}", Yraw, ref["raw"], ref["raw_bar"], RAW_EXACT)
    if want_act:
        est = _act_flip_estimate(ref, p, N)
        print(f"estimated share of Yact outputs __sinf may flip: {est:.5f}")
        _check(f"snake Yact {_ids(case)}", Yact, ref["act"], ref["act_bar"], ACT_EXACT)


def test_gemm_report_worst():
    """summary of the reference comparisons above (worst error / bar and lowest exact fraction per output kind)"""
    print({k: (round(v[0], 3), round(v[1], 5)) for k, v in WORST.items()})


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tiles(T, N, B):
    return -(-T // 128) * B * -(-N // 96)


@pytest.mark.parametrize("Cin", [96, 128])
def test_batch_rows_equal_single_sequence_runs(Cin):
    """each sequence of a KIND 0 batched launch equals its own KIND 1 single-sequence launch, bit for bit, with a
    causal dilated conv whose padding must come from that sequence alone"""
    T, N, taps, dil, B = 300, 960, 7, 3, 8
    assert _tiles(T, N, B) > _sms() * 3 // 2 >= _tiles(T, N, 1), "shape no longer selects KIND 0 / KIND 1"
    X, W, g = _inputs(B, T, Cin, N, taps, seed=Cin, x_std=2.0)
    p = _params(g, N, "bias res act", B, T)
    raw, act = debug_conv_gemm(X, W, dil=dil, act=True, **p)
    for b in range(B):
        pb = dict(p, R=p["R"][b:b + 1].contiguous())
        r1, a1 = debug_conv_gemm(X[b:b + 1].contiguous(), W, dil=dil, act=True, **pb)
        assert torch.equal(raw[b], r1[0]) and torch.equal(act[b], a1[0]), b


@pytest.mark.parametrize("T1", [5, 129])
def test_rows_do_not_depend_on_later_rows(T1):
    """output rows [0, T1) of a T = 300 run equal the T1 run (causality across M tiles)"""
    T2, Cin, N, taps, dil = 300, 64, 200, 7, 9
    X, W, g = _inputs(2, T2, Cin, N, taps, seed=T1)
    p = _params(g, N, "bias act", 2, T2)
    r2, a2 = debug_conv_gemm(X, W, dil=dil, act=True, **p)
    r1, a1 = debug_conv_gemm(X[:, :T1].contiguous(), W, dil=dil, act=True, **p)
    assert torch.equal(r2[:, :T1], r1) and torch.equal(a2[:, :T1], a1)


@pytest.mark.parametrize("mode,N1,N2", [(0, 8, 40), (0, 104, 200), (1, 32, 160), (1, 160, 1600)])
def test_columns_do_not_depend_on_later_weight_rows(mode, N1, N2):
    """the first N1 columns of an N2 run with the same first N1 weight rows equal the N1 run (N tails)"""
    T, Cin = 129, 96
    X, W, g = _inputs(1, T, Cin, N2, 1, seed=N1 + N2)
    kw = {}
    if mode == 0:
        kw = dict(bias=(torch.randn(N2, generator=g) * 0.5).cuda(), R=torch.randn(1, T, N2, generator=g).to(torch.bfloat16).cuda())
    r2, _ = debug_conv_gemm(X, W, mode=mode, **kw)
    if mode == 0:
        kw = dict(bias=kw["bias"][:N1].contiguous(), R=kw["R"][..., :N1].contiguous())
    r1, _ = debug_conv_gemm(X, W[:N1].contiguous(), mode=mode, **kw)
    n_out = N1 // 2 if mode == 1 else N1
    assert torch.equal(r2[..., :n_out], r1)


@pytest.mark.parametrize("taps,dil", [(7, 9), (2, 1)])
def test_history_rows_equal_one_shot_tail(taps, dil):
    """a run over [history ; new] with x_row0 = h equals rows [t0, t0 + T) of the one-shot run, bit for bit"""
    B, Tall, t0, Cin, N = 3, 300, 200, 64, 104
    X, W, g = _inputs(B, Tall, Cin, N, taps, seed=taps * dil)
    p = _params(g, N, "bias act", B, Tall)
    r_all, a_all = debug_conv_gemm(X, W, dil=dil, act=True, **p)
    h = (taps - 1) * dil
    Xs = X[:, t0 - h:].contiguous()
    r, a = debug_conv_gemm(Xs, W, dil=dil, T=Tall - t0, x_row0=h, history=True, act=True, **p)
    assert torch.equal(r, r_all[:, t0:]) and torch.equal(a, a_all[:, t0:])


def test_refusals_carry_the_kernel_message():
    """shapes and alignments the kernel does not take are refused with its own message, before any launch"""
    X, W, _ = _inputs(1, 16, 64, 64, 1, seed=1)
    with pytest.raises(EngineError, match=r"shape unsupported"):
        debug_conv_gemm(X[..., :48].contiguous(), W[..., :48].contiguous())            # Cin % 32
    with pytest.raises(EngineError, match=r"shape unsupported"):
        debug_conv_gemm(X, W[:12].contiguous())                                         # N % 8
    with pytest.raises(EngineError, match=r"shape unsupported"):
        debug_conv_gemm(X, W[:40].contiguous(), mode=1)                                 # SwiGLU N % 32
    buf = torch.zeros(16 * 64 + 8, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(EngineError, match=r"not 16-byte aligned"):
        debug_conv_gemm(buf[1:1 + 16 * 64].view(1, 16, 64), W)                          # X 2 bytes off
    torch.cuda.synchronize()
    r, _ = debug_conv_gemm(X, W)                                                        # the probe still works
    assert torch.isfinite(r.float()).all()
