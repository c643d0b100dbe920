"""float64 reference of the dense-layer GEMM shared by the prefill and the codec (fq3gemm::gemm, csrc/fq3_gemm.cuh),
and the per-element error bars its GPU test holds the kernel to.

    Y[t, n] = epilogue( sum_{tap, ci} W[n, tap, ci] * X[t - (taps-1-tap)*dil, ci] )

The sum is taken in float64; rows before a sequence's start (or outside [0, x_rows) with history rows) read as zero.
The epilogue rounds to bf16 (nearest even) at exactly the points the header lists:
    mode 0: v = rnd(acc + bias); v = v * scale; if R: v = rnd(rnd(v) + R) else v = rnd(v); Yact = rnd(v + ib sin^2(ea v))
    mode 1: Yraw[t, n/2] = rnd(rnd(silu(rnd(gate))) * rnd(up)) on (gate, up) = columns (2i, 2i + 1)
    mode 2: mode 0 with v = gelu_erf(rnd(acc + bias)), rounded again before the scale (the scale multiplies a bf16
            tensor, as in torch)

Bars.  The kernel accumulates bf16 products (exact in fp32) in fp32: wgmma adds one k16 chunk per instruction to the
fp32 accumulator, so an output sees K/16 accumulator roundings plus at most 16 inside a chunk.  Counting each as 2^-23
of sum|w x| (a rounding that truncates instead of rounding to nearest is still within one unit) bounds the accumulation
error by ACC_REL(K) * sum|w x|.  That error is carried through the epilogue by each stage's Lipschitz constant, and
every rounding point adds one bf16 ulp of its value (the kernel and the reference may round an input that differs by
the propagated error to neighbouring bf16 values), plus 2^-22 of the value for the fp32 arithmetic between rounding
points.  SnakeBeta also carries the error of __sinf: 2^-21.41 inside [-pi, pi] (CUDA C Programming Guide, intrinsic
functions); outside, the argument is reduced by a multiplication with 1/(2 pi) in fp32, which adds at most
|z| 2^-24 -- the bar uses |z| 2^-22.
"""
import math

import torch

GELU_LIP = 1.13      # max |d gelu(x) / dx| = 1.1289
SILU_LIP = 1.10      # max |d silu(x) / dx| = 1.0998
SIN_ERR_PI = 2.0 ** -21.41


def acc_rel(K: int) -> float:
    return (math.ceil(K / 16) + 16) * 2.0 ** -23


def rnd(x: torch.Tensor) -> torch.Tensor:
    """round float64 to bf16 (nearest even) and back to float64.  torch casts float64 to bf16 through float32, which
    rounds twice: 8.90625 + 3e-7 becomes the tie 8.90625 in float32 and then 8.875 instead of 8.9375.  Rounding to
    float32 toward zero with the last bit set when inexact ("round to odd") keeps the second rounding correct."""
    f = x.to(torch.float32)
    f = torch.where(f.to(torch.float64).abs() > x.abs(), torch.nextafter(f, torch.zeros_like(f)), f)
    odd = (f.to(torch.float64) != x).to(torch.int32)
    return (f.view(torch.int32) | odd).view(torch.float32).to(torch.bfloat16).to(torch.float64)


def ulp(x: torch.Tensor) -> torch.Tensor:
    """bf16 unit in the last place of |x| (8 significant bits)"""
    _, e = torch.frexp(x.abs().clamp(min=2.0 ** -126))
    return torch.ldexp(torch.ones_like(x), (e - 8).to(torch.int32))


def flip(v: torch.Tensor, err: torch.Tensor) -> torch.Tensor:
    """what one rounding point adds to a difference `err` in its input: one ulp plus the fp32 arithmetic before it"""
    m = v.abs() + err
    return ulp(m) + 2.0 ** -22 * m


def sin_err(z: torch.Tensor) -> torch.Tensor:
    return SIN_ERR_PI + z.abs() * 2.0 ** -22


def conv_acc(X: torch.Tensor, W: torch.Tensor, dil: int = 1, T=None, x_row0: int = 0, history: bool = False):
    """X [batch, rows, Cin], W [N, taps, Cin] -> (acc, sum|w x|), float64 [batch, T, N].
    Output row m of a sequence reads input row x_row0 + m - (taps-1-tap)*dil of that sequence, zero outside [0, rows).
    Without history rows: T = rows and x_row0 = 0."""
    if X.dim() == 2:
        X = X[None]
    B, rows, Cin = X.shape
    N, taps, _ = W.shape
    if not history:
        T, x_row0 = rows, 0
    Xd, Wd = X.to(torch.float64), W.to(torch.float64)
    acc = torch.zeros(B, T, N, dtype=torch.float64, device=X.device)
    mag = torch.zeros_like(acc)
    m = torch.arange(T, device=X.device)
    for tap in range(taps):
        src = x_row0 + m - (taps - 1 - tap) * dil
        ok = (src >= 0) & (src < rows)
        Xs = torch.zeros(B, T, Cin, dtype=torch.float64, device=X.device)
        Xs[:, ok] = Xd[:, src[ok]]
        acc += Xs @ Wd[:, tap].T
        mag += Xs.abs() @ Wd[:, tap].abs().T
    return acc, mag


def _col(p, N, device, default):
    """per-column parameter p[n % len(p)] as float64 [N]"""
    if p is None:
        return torch.full((N,), float(default), dtype=torch.float64, device=device)
    p = p.to(device=device, dtype=torch.float64).reshape(-1)
    return p[torch.arange(N, device=device) % p.numel()]


def epilogue(acc, mag, K: int, mode: int = 0, bias=None, scale=None, R=None, ea=None, ib=None, act: bool = False):
    """The kernel's epilogue in float64 with bf16 rounding points.  Returns dict(raw, raw_bar[, act, act_bar]): values
    are float64 tensors holding bf16 values, bars are per-element bounds on |kernel - reference|."""
    d = acc_rel(K) * mag
    if mode == 1:
        g, u, dg, du = acc[..., 0::2], acc[..., 1::2], d[..., 0::2], d[..., 1::2]
        rg, eg = rnd(g), dg + flip(g, dg)
        ru, eu = rnd(u), du + flip(u, du)
        s = rg * torch.sigmoid(rg)
        rs = rnd(s)
        es = SILU_LIP * eg + flip(s, SILU_LIP * eg)
        out = rs * ru
        e = ru.abs() * es + rs.abs() * eu + es * eu
        return dict(raw=rnd(out), raw_bar=e + flip(out, e))
    N = acc.shape[-1]
    v = acc + _col(bias, N, acc.device, 0.0)
    e = d + flip(v, d)
    v = rnd(v)
    exact = True     # v is still a bf16 value: rounding it again adds nothing
    if mode == 2:
        # the kernel's 0.5 x (1 + erff(x / sqrt 2)) in fp32 is off by up to |x| 2^-23 in absolute terms where 1 + erf
        # cancels (x < -4); the relative 2^-22 of flip() does not cover that tail
        e, exact = GELU_LIP * e + v.abs() * 2.0 ** -22, False
        v = 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0)))
    if scale is not None:
        if not exact:
            e = e + flip(v, e)
        s = _col(scale, N, acc.device, 1.0)
        v, e, exact = rnd(v) * s, e * s.abs(), False
    if R is not None:
        if not exact:
            e = e + flip(v, e)
        v, exact = rnd(v) + R.to(torch.float64), False
    if not exact:
        e = e + flip(v, e)
    raw = rnd(v)
    out = dict(raw=raw, raw_bar=e)
    if act:
        a, b = _col(ea, N, acc.device, 1.0), _col(ib, N, acc.device, 0.0)
        z = a * raw
        y = raw + b * torch.sin(z) ** 2
        ea_ = (1.0 + b * a) * e + 2.0 * b * sin_err(z)
        out["act"] = rnd(y)
        out["act_bar"] = ea_ + flip(y, ea_)
    return out
