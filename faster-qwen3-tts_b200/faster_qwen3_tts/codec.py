"""Codec decoder (RVQ codes -> 24 kHz PCM) behind the ``speech_tokenizer.decode`` contract the reference calls
(model.py:924,1093,1122; tests/test_sample_rate.py:53-75):

    speech_tokenizer.decode({"audio_codes": LongTensor[1, T, 16]}) -> ([wav Tensor[1920*T]], 24000)

The real Qwen3-TTS tokenizer decoder ships inside the absent ``qwen-tts`` package; its geometry is restated from the
in-image analogue ``transformers/models/qwen3_omni_moe/modeling_qwen3_omni_moe.py`` (Code2Wav :3730-3790, causal
convs :3283-3330, ConvNeXt :3333-3366, SnakeBeta :3645-3683, decoder block :3705-3727, pre-transformer :3370-3640):
16-codebook embedding mean -> 8-layer sliding-window pre-transformer (H=1024) -> 2x(ConvTranspose k=2,s=2 + ConvNeXt)
-> conv7 1024->1536 -> 4 blocks [SnakeBeta, causal ConvTranspose (k=2r, s=r), 3 residual units (SnakeBeta, dilated
conv7, SnakeBeta, conv1)] with r = 8,5,4,3 and channels 1536->768->384->192->96 -> SnakeBeta -> conv7 -> clamp.
Total upsample 1920.  "parity unpinned" (analogue geometry, synthetic weights).

The torch module below is the weight container and the library (cuDNN / cuBLAS) functional baseline
(``backend="torch"``).  ``backend="engine"`` -- the default on CUDA -- runs the WHOLE decode, codes in / PCM out, in
the hand-written sm_90a kernels behind the C ABI (``fq3_codec_decode_codes``, csrc/fq3_codec.cu): no library kernel
is launched (DESIGN.md, kernel K4).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F


@dataclass
class Code2WavConfig:
    codebook_size: int = 2048
    num_quantizers: int = 16
    hidden_size: int = 1024
    num_hidden_layers: int = 8
    num_attention_heads: int = 16
    intermediate_size: int = 3072
    sliding_window: int = 72
    rms_norm_eps: float = 1e-5
    layer_scale: float = 0.01
    rope_theta: float = 10000.0
    upsampling_ratios: Tuple[int, ...] = (2, 2)
    upsample_rates: Tuple[int, ...] = (8, 5, 4, 3)
    decoder_dim: int = 1536
    sample_rate: int = 24000

    @property
    def total_upsample(self) -> int:
        return int(math.prod(self.upsampling_ratios) * math.prod(self.upsample_rates))


def tiny_codec_config() -> Code2WavConfig:
    return Code2WavConfig(codebook_size=64, hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                          intermediate_size=256, sliding_window=8, decoder_dim=64)


class CausalConv1d(nn.Module):
    def __init__(self, cin, cout, k, dilation=1, groups=1):
        super().__init__()
        self.conv = nn.Conv1d(cin, cout, k, dilation=dilation, groups=groups)
        self.pad = (k - 1) * dilation

    def forward(self, x):
        return self.conv(F.pad(x, (self.pad, 0)))


class CausalConvTranspose1d(nn.Module):
    def __init__(self, cin, cout, k, stride):
        super().__init__()
        self.conv = nn.ConvTranspose1d(cin, cout, k, stride=stride)
        self.trim = k - stride

    def forward(self, x):
        y = self.conv(x)  # length (T-1)*s + k; dropping the k-s tail keeps it causal and exactly T*s long
        return y[..., : y.shape[-1] - self.trim] if self.trim else y


class SnakeBeta(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.alpha = nn.Parameter(torch.zeros(c))
        self.beta = nn.Parameter(torch.zeros(c))

    def forward(self, x):
        a = torch.exp(self.alpha)[None, :, None]
        b = torch.exp(self.beta)[None, :, None]
        return x + (1.0 / (b + 1e-9)) * torch.sin(x * a).pow(2)


class ConvNeXt(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.dwconv = CausalConv1d(c, c, 7, groups=c)
        self.norm = nn.LayerNorm(c, eps=1e-6)
        self.pwconv1 = nn.Linear(c, 4 * c)
        self.pwconv2 = nn.Linear(4 * c, c)
        self.gamma = nn.Parameter(1e-6 * torch.ones(c))

    def forward(self, x):
        h = self.dwconv(x).transpose(1, 2)
        h = self.pwconv2(F.gelu(self.pwconv1(self.norm(h))))
        return x + (self.gamma * h).transpose(1, 2)


class ResidualUnit(nn.Module):
    def __init__(self, c, dilation):
        super().__init__()
        self.act1, self.conv1 = SnakeBeta(c), CausalConv1d(c, c, 7, dilation=dilation)
        self.act2, self.conv2 = SnakeBeta(c), CausalConv1d(c, c, 1)

    def forward(self, x):
        return x + self.conv2(self.act2(self.conv1(self.act1(x))))


class DecoderBlock(nn.Module):
    def __init__(self, cin, cout, rate):
        super().__init__()
        self.act = SnakeBeta(cin)
        self.up = CausalConvTranspose1d(cin, cout, 2 * rate, rate)
        self.res = nn.ModuleList([ResidualUnit(cout, d) for d in (1, 3, 9)])

    def forward(self, x):
        x = self.up(self.act(x))
        for r in self.res:
            x = r(x)
        return x


class _RMS(nn.Module):
    def __init__(self, n, eps):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(n))
        self.eps = eps

    def forward(self, x):
        dt = x.dtype
        xf = x.float()
        return self.weight * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + self.eps)).to(dt)


class PreLayer(nn.Module):
    def __init__(self, c: Code2WavConfig):
        super().__init__()
        H, I = c.hidden_size, c.intermediate_size
        self.nh = c.num_attention_heads
        self.q, self.k, self.v, self.o = (nn.Linear(H, H, bias=False) for _ in range(4))
        self.gate, self.up, self.down = nn.Linear(H, I, bias=False), nn.Linear(H, I, bias=False), nn.Linear(I, H, bias=False)
        self.ln1, self.ln2 = _RMS(H, c.rms_norm_eps), _RMS(H, c.rms_norm_eps)
        self.s1 = nn.Parameter(torch.full((H,), c.layer_scale))
        self.s2 = nn.Parameter(torch.full((H,), c.layer_scale))

    def forward(self, x, cos, sin, mask):
        B, T, H = x.shape
        hd = H // self.nh
        h = self.ln1(x)
        q = self.q(h).view(B, T, self.nh, hd).transpose(1, 2)
        k = self.k(h).view(B, T, self.nh, hd).transpose(1, 2)
        v = self.v(h).view(B, T, self.nh, hd).transpose(1, 2)

        def rot(t):
            a, b = t[..., : hd // 2], t[..., hd // 2:]
            return torch.cat((-b, a), dim=-1)

        q = q * cos + rot(q) * sin
        k = k * cos + rot(k) * sin
        o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask)
        x = x + self.s1 * self.o(o.transpose(1, 2).reshape(B, T, H))
        h = self.ln2(x)
        return x + self.s2 * self.down(F.silu(self.gate(h)) * self.up(h))


class Code2Wav(nn.Module):
    def __init__(self, c: Code2WavConfig):
        super().__init__()
        self.config = c
        H = c.hidden_size
        self.code_embedding = nn.Embedding(c.codebook_size * c.num_quantizers, H)
        self.layers = nn.ModuleList([PreLayer(c) for _ in range(c.num_hidden_layers)])
        self.norm = _RMS(H, c.rms_norm_eps)
        self.upsample = nn.ModuleList([nn.ModuleList([CausalConvTranspose1d(H, H, r, r), ConvNeXt(H)])
                                       for r in c.upsampling_ratios])
        self.conv_in = CausalConv1d(H, c.decoder_dim, 7)
        chans = [c.decoder_dim // (2 ** i) for i in range(len(c.upsample_rates) + 1)]
        self.blocks = nn.ModuleList([DecoderBlock(chans[i], chans[i + 1], r) for i, r in enumerate(c.upsample_rates)])
        self.act_out = SnakeBeta(chans[-1])
        self.conv_out = CausalConv1d(chans[-1], 1, 7)

    def forward(self, codes: torch.Tensor) -> torch.Tensor:
        """codes [B, Q, T] -> wav [B, 1, 1920*T] clamped to [-1, 1]."""
        c = self.config
        B, Q, T = codes.shape
        off = (torch.arange(Q, device=codes.device) * c.codebook_size).view(1, Q, 1)
        x = self.code_embedding(codes + off).mean(1)  # [B,T,H]
        hd = c.hidden_size // c.num_attention_heads
        inv = 1.0 / (c.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.float32, device=x.device) / hd))
        fr = torch.arange(T, dtype=torch.float32, device=x.device)[:, None] * inv[None]
        emb = torch.cat((fr, fr), dim=-1)
        cos, sin = emb.cos().to(x.dtype)[None, None], emb.sin().to(x.dtype)[None, None]
        i = torch.arange(T, device=x.device)
        allowed = (i[None, :] <= i[:, None]) & (i[None, :] > i[:, None] - c.sliding_window)
        for l in self.layers:
            x = l(x, cos, sin, allowed)
        x = self.norm(x).transpose(1, 2)
        for up, nx in self.upsample:
            x = nx(up(x))
        x = self.conv_in(x)
        for b in self.blocks:
            x = b(x)
        return self.conv_out(self.act_out(x)).clamp(-1, 1)


class SpeechTokenizer:
    """The decode side of the upstream speech tokenizer, as the reference consumes it
    (``decode({"audio_codes": [B,T,16]}) -> ([wav], sample_rate)``).

    backend="engine": codes -> PCM entirely in the hand-written sm_90a kernels of csrc/fq3_codec.cu through the C
    ABI: front end (code-embedding mean, 8-layer sliding-window pre-transformer, 2 x (ConvTranspose k=2 + ConvNeXt))
    and waveform stack (conv_in, 4 upsampling blocks, conv_out) -- ``fq3_codec_decode_codes``.
    backend="torch": the plain library implementation."""

    def __init__(self, decoder: Code2Wav, backend: str = "torch"):
        self.decoder = decoder
        self.sample_rate = decoder.config.sample_rate
        self.launches = 0
        self.backend = backend
        self._h = None
        self._stream_pool = []      # released stream handles: a request re-uses one (async reset) instead of cudaMalloc / cudaFree
        self._ref_templates = {}    # content hash of a voice reference's codes -> stream warmed with them (bounded)
        if backend == "engine":
            self._init_engine()
            self._init_frontend()

    # ---- engine plumbing -------------------------------------------------------------------------------
    def _init_engine(self):
        import ctypes as C
        from .engine import Tensor, load_library
        lib = load_library()
        d = self.decoder
        c = d.config
        p0 = next(d.parameters())
        if p0.device.type != "cuda":
            raise RuntimeError("codec engine backend needs the decoder on a CUDA device")
        self._lib, self._dev = lib, p0.device
        geom = [p0.device.index or 0, c.hidden_size, c.decoder_dim, len(c.upsample_rates)] + list(c.upsample_rates)
        arr = (C.c_int32 * len(geom))(*geom)
        h = C.c_void_p()
        if lib.fq3_codec_create(arr, len(geom), C.byref(h)):
            raise RuntimeError(lib.fq3_codec_last_error().decode())
        t = {}

        def put(name, x):
            t[name] = x.detach().to(torch.float32).contiguous()

        put("conv_in.w", d.conv_in.conv.weight); put("conv_in.b", d.conv_in.conv.bias)
        for i, b in enumerate(d.blocks):
            put(f"b{i}.act.a", b.act.alpha); put(f"b{i}.act.b", b.act.beta)
            put(f"b{i}.up.w", b.up.conv.weight); put(f"b{i}.up.b", b.up.conv.bias)
            for j, r in enumerate(b.res):
                q = f"b{i}.r{j}"
                put(q + ".a1.a", r.act1.alpha); put(q + ".a1.b", r.act1.beta)
                put(q + ".c1.w", r.conv1.conv.weight); put(q + ".c1.b", r.conv1.conv.bias)
                put(q + ".a2.a", r.act2.alpha); put(q + ".a2.b", r.act2.beta)
                put(q + ".c2.w", r.conv2.conv.weight); put(q + ".c2.b", r.conv2.conv.bias)
        put("out.act.a", d.act_out.alpha); put("out.act.b", d.act_out.beta)
        put("out.w", d.conv_out.conv.weight); put("out.b", d.conv_out.conv.bias)
        arr_t = (Tensor * len(t))()
        for i, (k, v) in enumerate(t.items()):
            arr_t[i] = Tensor(k.encode(), v.data_ptr(), v.numel())
        with torch.cuda.device(self._dev):
            if lib.fq3_codec_load_weights(h, arr_t, len(t), C.c_void_p(torch.cuda.current_stream(self._dev).cuda_stream)):
                raise RuntimeError(lib.fq3_codec_last_error().decode())
        self._h = h

    def _init_frontend(self):
        import ctypes as C
        from .engine import Tensor
        d, lib = self.decoder, self._lib
        c = d.config
        t = {}

        def put(name, x):
            t[name] = x.detach().to(torch.float32).contiguous()

        put("fe.embed", d.code_embedding.weight)
        put("fe.norm", d.norm.weight)
        for i, l in enumerate(d.layers):
            p = f"fe.l{i}"
            put(p + ".ln1", l.ln1.weight); put(p + ".ln2", l.ln2.weight); put(p + ".s1", l.s1); put(p + ".s2", l.s2)
            put(p + ".q", l.q.weight); put(p + ".k", l.k.weight); put(p + ".v", l.v.weight); put(p + ".o", l.o.weight)
            put(p + ".gate", l.gate.weight); put(p + ".up", l.up.weight); put(p + ".down", l.down.weight)
        for i, (up, nx) in enumerate(d.upsample):
            p = f"fe.u{i}"
            put(p + ".ct.w", up.conv.weight); put(p + ".ct.b", up.conv.bias)
            put(p + ".dw.w", nx.dwconv.conv.weight); put(p + ".dw.b", nx.dwconv.conv.bias)
            put(p + ".ln.w", nx.norm.weight); put(p + ".ln.b", nx.norm.bias)
            put(p + ".pw1.w", nx.pwconv1.weight); put(p + ".pw1.b", nx.pwconv1.bias)
            put(p + ".pw2.w", nx.pwconv2.weight); put(p + ".pw2.b", nx.pwconv2.bias)
            put(p + ".gamma", nx.gamma)
        geom = [c.num_quantizers, c.codebook_size, c.hidden_size, c.intermediate_size, c.num_attention_heads,
                c.num_hidden_layers, c.sliding_window, len(c.upsampling_ratios)] + list(c.upsampling_ratios)
        g = (C.c_int32 * len(geom))(*geom)
        fg = (C.c_float * 2)(c.rms_norm_eps, c.rope_theta)
        arr_t = (Tensor * len(t))()
        for i, (k, v) in enumerate(t.items()):
            arr_t[i] = Tensor(k.encode(), v.data_ptr(), v.numel())
        with torch.cuda.device(self._dev):
            if lib.fq3_codec_load_frontend(self._h, g, len(geom), fg, 2, arr_t, len(t),
                                           C.c_void_p(torch.cuda.current_stream(self._dev).cuda_stream)):
                raise RuntimeError(lib.fq3_codec_last_error().decode())
            torch.cuda.current_stream(self._dev).synchronize()

    def __del__(self):
        try:
            if self._h is not None:
                for t in list(self._ref_templates.values()):
                    t.close()
                self._ref_templates = {}
                for h in self._stream_pool:
                    self._lib.fq3_codec_stream_destroy(h)
                self._stream_pool = []
                self._lib.fq3_codec_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def _engine_call(self, codes: torch.Tensor, want_pcm: bool, call):
        """What every engine codec call shares: codes [B, n, Q] as int64 on the codec's device, the code-group check, the
        PCM buffer, the device context and the error check.  ``call(codes_ptr, B, n, pcm_ptr, stream)`` makes the C ABI
        call (pcm_ptr None without PCM).  Returns the B PCM rows, or None."""
        import ctypes as C
        codes = codes.to(device=self._dev, dtype=torch.long).contiguous()
        B, n, Q = codes.shape
        if Q != self.decoder.config.num_quantizers:
            raise ValueError(f"audio_codes must have {self.decoder.config.num_quantizers} code groups, got {Q}")
        pcm = torch.empty(B, n * self.decoder.config.total_upsample, dtype=torch.float32, device=self._dev) if want_pcm else None
        with torch.cuda.device(self._dev):
            rc = call(C.c_void_p(codes.data_ptr()), B, n, C.c_void_p(pcm.data_ptr()) if want_pcm else None,
                      C.c_void_p(torch.cuda.current_stream(self._dev).cuda_stream))
        if rc:
            raise RuntimeError(self._lib.fq3_codec_last_error().decode())
        self.launches = int(self._lib.fq3_codec_launch_count(self._h))
        return [pcm[b] for b in range(B)] if want_pcm else None

    @torch.inference_mode()
    def decode(self, payload) -> Tuple[List[torch.Tensor], int]:
        codes = payload["audio_codes"]  # [B, T, Q]
        if self.backend == "engine":
            pcm = self._engine_call(codes, True, lambda *a: self._lib.fq3_codec_decode_codes(self._h, *a))
            return pcm, self.sample_rate
        dev = next(self.decoder.parameters()).device
        wav = self.decoder(codes.to(dev).transpose(1, 2).contiguous())
        self.launches += 1
        return [w.reshape(-1).float() for w in wav], self.sample_rate

    # ---- stateful streaming (fq3_codec_stream_*) -----------------------------------------------------------
    @property
    def supports_streams(self) -> bool:
        """decoder streams exist only on the engine codec"""
        return self.backend == "engine" and self._h is not None

    def open_stream(self) -> "CodecStream":
        """A decoder stream that keeps every causal layer's history on the device: ``push(codes[n,16])`` returns the
        1920*n samples of exactly those frames, at the cost of n frames (no window re-decode)."""
        if not self.supports_streams:
            raise RuntimeError("stateful streaming needs the engine backend")
        return CodecStream(self)

    def clear_reference_cache(self) -> None:
        """forget the warmed template streams (a new speaker pays one decode of its reference again)"""
        for t in list(self._ref_templates.values()):
            t.close()
        self._ref_templates = {}

    @torch.inference_mode()
    def reference_stream(self, ref_codes: torch.Tensor, create: bool = True) -> Optional["CodecStream"]:
        """A stream whose state is "these reference frames have been decoded": the first request with a reference warms
        a template (one decode of the reference), every later one gets a device-to-device copy of it -- the codec-side
        counterpart of the reference's voice-prompt cache (model.py:415-463).  ``create=False``: None when no template
        exists for this reference yet (the caller decides when to pay for the warm-up)."""
        import ctypes as C
        import hashlib
        rc = ref_codes.detach().to(torch.long).cpu().contiguous()
        key = (tuple(rc.shape), hashlib.blake2b(rc.numpy().tobytes(), digest_size=16).digest())
        tpl = self._ref_templates.get(key)
        if tpl is None and not create:
            return None
        if tpl is None:
            tpl = self.open_stream()
            tpl.warm(ref_codes)
            if len(self._ref_templates) >= 16:
                self._ref_templates.pop(next(iter(self._ref_templates))).close()
            self._ref_templates[key] = tpl
        s = self.open_stream()
        with torch.cuda.device(self._dev):
            if self._lib.fq3_codec_stream_copy(s._h, tpl._h, C.c_void_p(torch.cuda.current_stream(self._dev).cuda_stream)):
                raise RuntimeError(self._lib.fq3_codec_last_error().decode())
        return s

    @torch.inference_mode()
    def push_streams(self, streams, codes: torch.Tensor, want_pcm: bool = True):
        """The next n frames of several streams in ONE set of launches: codes [B, n, 16] -> list of B PCM tensors
        (or None with want_pcm=False: state warm-up, e.g. the ICL reference frames)."""
        import ctypes as C
        if codes.shape[0] != len(streams):
            raise ValueError("one row of codes per stream")
        arr = (C.c_void_p * len(streams))(*[s._h for s in streams])
        return self._engine_call(codes, want_pcm, lambda codes_p, B, n, pcm_p, stream:
                                 self._lib.fq3_codec_stream_decode(self._h, arr, B, codes_p, n, pcm_p, stream))

    def flops(self, T: int) -> float:
        """dense-layer FLOPs of the waveform stack for T code frames"""
        return float(self._lib.fq3_codec_flops(self._h, 4 * T)) if self._h is not None else 0.0

    def frontend_flops(self, T: int) -> float:
        return float(self._lib.fq3_codec_frontend_flops(self._h, T)) if self._h is not None else 0.0


class CodecStream:
    """One stateful decoder stream (C ABI fq3_codec_stream_*): history of every causal layer lives on the device.
    Handles are pooled by the tokenizer: opening a stream for a new request re-uses a released one (asynchronous reset of
    its 3.8 MB state) -- no cudaMalloc / cudaFree, and none of their device-wide synchronisation, on the request path."""

    def __init__(self, st: SpeechTokenizer):
        import ctypes as C
        self.st = st
        if st._stream_pool:
            self._h = st._stream_pool.pop()
            self.reset()
            return
        h = C.c_void_p()
        with torch.cuda.device(st._dev):
            if st._lib.fq3_codec_stream_create(st._h, C.byref(h)):
                raise RuntimeError(st._lib.fq3_codec_last_error().decode())
        self._h = h

    @property
    def frames(self) -> int:
        return int(self.st._lib.fq3_codec_stream_frames(self._h))

    def push(self, codes: torch.Tensor) -> torch.Tensor:
        """codes [n,16] -> PCM float32 [1920*n] of exactly these frames"""
        return self.st.push_streams([self], codes.reshape(1, -1, codes.shape[-1]))[0]

    def warm(self, codes: torch.Tensor) -> None:
        """feed frames whose audio is not wanted (the ICL reference): state only"""
        self.st.push_streams([self], codes.reshape(1, -1, codes.shape[-1]), want_pcm=False)

    def reset(self) -> None:
        import ctypes as C
        with torch.cuda.device(self.st._dev):
            self.st._lib.fq3_codec_stream_reset(self._h, C.c_void_p(torch.cuda.current_stream(self.st._dev).cuda_stream))

    def close(self) -> None:
        """hand the stream back to the tokenizer's pool"""
        if self._h is not None and self.st._h is not None:
            self.st._stream_pool.append(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def build_codec(cfg: Code2WavConfig = None, seed: int = 0, dtype=torch.bfloat16, device="cpu",
                backend: str = None) -> SpeechTokenizer:
    cfg = cfg or Code2WavConfig()
    dev = torch.device(device)
    if backend is None:
        backend = "engine" if dev.type == "cuda" else "torch"
    with torch.device(dev):
        m = Code2Wav(cfg)
    g = torch.Generator(device=dev).manual_seed(seed)
    for name, p in m.named_parameters():
        p.requires_grad_(False)
        if name.endswith(("alpha", "beta")):
            p.normal_(0.0, 0.3, generator=g)
        elif name.endswith("gamma"):
            p.fill_(0.1)
        elif ".s1" in name or ".s2" in name:
            pass
        elif p.dim() == 1 and ("ln" in name or "norm" in name) and name.endswith("weight"):
            p.fill_(1.0)
        elif p.dim() == 1:
            p.normal_(0.0, 0.01, generator=g)
        elif "code_embedding" in name:
            p.normal_(0.0, 1.0, generator=g)
        else:
            fan_in = p[0].numel()
            p.normal_(0.0, 0.5 / math.sqrt(fan_in), generator=g)
    return SpeechTokenizer(m.to(dtype=dtype), backend=backend)
