"""The float64 reference of the dense-layer GEMM (tests/util_gemm.py) checked on its own, so that the GPU test compares
the kernel with something known to be right: its convolution against F.conv1d, its history-row addressing against the
one-shot result, and its rounding points against the torch bf16 expressions the kernel header names."""
import pytest
import torch
import torch.nn.functional as F

from util_gemm import conv_acc, epilogue, rnd, ulp


def _data(B, T, Cin, N, taps, seed):
    g = torch.Generator().manual_seed(seed)
    X = torch.randn(B, T, Cin, generator=g).to(torch.bfloat16)
    W = (torch.randn(N, taps, Cin, generator=g) * 0.2).to(torch.bfloat16)
    return X, W


@pytest.mark.parametrize("taps,dil,T,B", [(1, 1, 5, 1), (2, 1, 7, 2), (7, 1, 20, 1), (7, 3, 9, 2), (7, 9, 40, 3),
                                          (3, 9, 5, 1)])
def test_conv_matches_conv1d(taps, dil, T, B):
    """causal dilated conv1d with explicit left padding, per sequence (shifts up to 54 > T included)"""
    X, W = _data(B, T, 32, 24, taps, seed=taps * 100 + dil * 10 + T)
    acc, mag = conv_acc(X, W, dil)
    x = F.pad(X.double().permute(0, 2, 1), ((taps - 1) * dil, 0))
    want = F.conv1d(x, W.double().permute(0, 2, 1), dilation=dil).permute(0, 2, 1)
    assert acc.shape == (B, T, 24)
    torch.testing.assert_close(acc, want, rtol=1e-12, atol=1e-12)
    want_mag = F.conv1d(x.abs(), W.double().abs().permute(0, 2, 1), dilation=dil).permute(0, 2, 1)
    torch.testing.assert_close(mag, want_mag, rtol=1e-12, atol=1e-12)
    # sequences do not see each other: the conv of sequence b alone
    for b in range(B):
        torch.testing.assert_close(conv_acc(X[b:b + 1], W, dil)[0], acc[b:b + 1], rtol=0, atol=0)


@pytest.mark.parametrize("taps,dil,h_extra", [(7, 3, 0), (7, 9, 5), (2, 1, 0), (1, 1, 3)])
def test_history_rows_equal_one_shot_tail(taps, dil, h_extra):
    """[history ; new] with x_row0 = h rows of history reproduces rows [t0, t0 + Tn) of the one-shot conv; history rows
    beyond what the receptive field needs change nothing, and missing ones read as zero like the causal padding"""
    B, T, Tn, t0 = 2, 90, 11, 70
    X, W = _data(B, T, 64, 16, taps, seed=7 + taps + dil)
    one_shot, _ = conv_acc(X, W, dil)
    h = (taps - 1) * dil + h_extra
    Xs = X[:, t0 - h:t0 + Tn].contiguous()
    got, _ = conv_acc(Xs, W, dil, T=Tn, x_row0=h, history=True)
    torch.testing.assert_close(got, one_shot[:, t0:t0 + Tn], rtol=1e-12, atol=1e-12)
    # a stream at its very start: no history rows exist yet, so the one-shot head
    got0, _ = conv_acc(X[:, :Tn].contiguous(), W, dil, T=Tn, x_row0=0, history=True)
    torch.testing.assert_close(got0, one_shot[:, :Tn], rtol=1e-12, atol=1e-12)


def test_rounding_points_match_torch_bf16_expressions():
    """each epilogue equals the torch bf16 eager expression of the layer it fuses"""
    g = torch.Generator().manual_seed(3)
    acc = torch.randn(2, 9, 64, generator=g, dtype=torch.float64) * 3
    mag = torch.zeros_like(acc)
    bias = torch.randn(16, generator=g)
    scale = torch.rand(64, generator=g) + 0.1
    R = torch.randn(2, 9, 64, generator=g).to(torch.bfloat16)
    bcol = bias.double()[torch.arange(64) % 16]
    # mode 0: Linear(bias) -> * gamma -> + residual, every op a bf16 tensor in torch
    lin = (acc + bcol).float().to(torch.bfloat16)
    want = (lin.float() * scale).to(torch.bfloat16) + R
    got = epilogue(acc, mag, 64, 0, bias=bias, scale=scale, R=R)
    assert torch.equal(got["raw"], want.double())
    # mode 2: GELU(Linear) in bf16, the GELU itself evaluated in float64 (torch's and the kernel's fp32 formula lose
    # their relative accuracy in the far negative tail, where 1 + erf cancels)
    got = epilogue(acc, mag, 64, 2, bias=bias)
    assert torch.equal(got["raw"], F.gelu(lin.double()).to(torch.bfloat16).double())
    # mode 1: silu(gate) * up in bf16
    got = epilogue(acc, mag, 64, 1)
    gate, up = acc[..., 0::2].float().to(torch.bfloat16), acc[..., 1::2].float().to(torch.bfloat16)
    assert torch.equal(got["raw"], (F.silu(gate) * up).double())
    # SnakeBeta on the rounded raw value
    ea, ib = torch.rand(64, generator=g) + 0.5, torch.rand(64, generator=g) + 0.5
    got = epilogue(acc, mag, 64, 0, bias=bias, ea=ea, ib=ib, act=True)
    x = got["raw"]
    assert torch.equal(got["act"], rnd(x + ib.double() * torch.sin(ea.double() * x) ** 2))
    # with no accumulation error and no later arithmetic the bar is exactly the ulp of each rounding point
    got = epilogue(acc, mag, 64, 0)
    assert torch.allclose(got["raw_bar"], ulp(acc.abs()) + 2.0 ** -22 * acc.abs())


def test_rnd_rounds_float64_once():
    """correct rounding from float64, where torch's cast through float32 would round twice"""
    x = torch.tensor([8.90625 + 3e-7, 8.90625, 8.90625 - 3e-7, -8.90625 - 3e-7, 1.0 + 2.0 ** -8, 1.0 + 2.0 ** -8 + 1e-12,
                      3.0, 0.0], dtype=torch.float64)
    assert rnd(x).tolist() == [8.9375, 8.875, 8.875, -8.9375, 1.0, 1.0 + 2.0 ** -7, 3.0, 0.0]
    g = torch.Generator().manual_seed(0)
    y = torch.randn(10000, generator=g, dtype=torch.float64) * 100
    assert ((rnd(y) - y).abs() <= ulp(y) / 2).all()


def test_ulp():
    x = torch.tensor([1.0, 1.5, 2.0, -3.0, 0.75, 256.0], dtype=torch.float64)
    assert ulp(x).tolist() == [2 ** -7, 2 ** -7, 2 ** -6, 2 ** -6, 2 ** -8, 2.0]
