"""PCM bar of BASELINE.json's north_star: "output audio matches the reference on fixed seeds within 1e-3 max-abs PCM".

The engine's codec path (`speech_tokenizer.decode`, C ABI `fq3_codec_decode_codes`) against the fp32
ORACLE decode held under oracle/ (oracle/codec_oracle.py, pinned to the Hugging Face Code2Wav analogue on CPU), same
weights, same codes, at the FULL decoder geometry (1536 -> 96 channels, rates 8*5*4*3) and at the two window lengths the
streaming policy produces (model.py:1085-1135): Phase 2 = 25 context + 8 new frames (T=33), Phase 1 with an ICL
reference = 174 + 8 frames (T=182).  Tolerance 1e-3 max-abs, as north_star states."""
import pytest
import torch

from oracle import codec_oracle

pytestmark = pytest.mark.gpu

TOL = 1e-3


@pytest.fixture(scope="module")
def full_codec():
    from faster_qwen3_tts.codec import Code2WavConfig, build_codec
    cfg = Code2WavConfig()
    assert cfg.decoder_dim == 1536 and tuple(cfg.upsample_rates) == (8, 5, 4, 3)
    return build_codec(cfg, seed=3, dtype=torch.bfloat16, device="cuda", backend="engine")


def _oracle(st, codes):
    c = st.decoder.config
    with torch.inference_mode():
        return codec_oracle.decode(st.decoder.state_dict(), codes, codebook_size=c.codebook_size,
                                   num_attention_heads=c.num_attention_heads, sliding_window=c.sliding_window,
                                   rms_norm_eps=c.rms_norm_eps, rope_theta=c.rope_theta,
                                   upsampling_ratios=c.upsampling_ratios, upsample_rates=c.upsample_rates)


@pytest.mark.parametrize("T", [33, 182, 8, 5, 100])
def test_full_geometry_window_pcm_within_1e3_of_fp32_oracle(full_codec, T):
    st = full_codec
    codes = torch.randint(0, 2048, (T, 16), generator=torch.Generator().manual_seed(T), device="cpu").cuda()
    got, sr = st.decode({"audio_codes": codes[None]})
    want = _oracle(st, codes)
    assert sr == 24000 and got[0].shape[0] == 1920 * T == want.shape[0]
    err = (got[0] - want).abs().max().item()
    peak, rms = want.abs().max().item(), want.pow(2).mean().sqrt().item()
    # yardstick: the same bf16 weights through the torch / cuDNN modules (the arithmetic the reference itself executes)
    with torch.inference_mode():
        lib16 = st.decoder(codes.t()[None])[0, 0].float()
    err_lib = (lib16 - want).abs().max().item()
    print(f"T={T}: max|engine - fp32 oracle| = {err:.3e}  max|torch bf16 modules - fp32 oracle| = {err_lib:.3e}  "
          f"(oracle peak {peak:.3f}, rms {rms:.4f})")
    assert peak > 0.02            # a real signal reaches the output
    assert err < TOL
    assert err < 1.5 * err_lib + 1e-5   # bf16 arithmetic costs the hand-written path no more than the library path


def test_streaming_windows_end_to_end_codes_to_pcm(full_codec):
    """codes -> PCM through the reference's window policy (ICL reference of 174 frames, chunk 8): every emitted chunk
    against the oracle decoding the same window with the same trim."""
    from faster_qwen3_tts.model import _StreamWindow
    import types
    st = full_codec
    g = torch.Generator().manual_seed(5)
    ref = torch.randint(0, 2048, (174, 16), generator=g).cuda()
    owner = types.SimpleNamespace(_to_numpy=None)
    win = _StreamWindow(owner, st, ref, 8, to_host=False)
    gen = []
    worst = 0.0
    for ci in range(6):
        chunk = torch.randint(0, 2048, (8, 16), generator=g).cuda()
        gen.append(chunk)
        audio, sr = win.push(chunk)
        flat = torch.cat(gen)
        n_total = flat.shape[0]
        if ci < 4:      # Phase 1 (fewer than 25 generated frames before this chunk completes calibration at 32)
            inp = torch.cat([ref, flat])
            full = _oracle(st, inp)
            cut = int(174 / inp.shape[0] * full.shape[0])
            want = full[cut:][(n_total - 8) * 1920:]
        else:           # Phase 2: 25 context frames + the 8 new ones
            window = flat[n_total - 8 - 25:]
            want = _oracle(st, window)[25 * 1920:]
        assert audio.shape[0] == want.shape[0] == 8 * 1920, (ci, audio.shape, want.shape)
        err = (audio - want).abs().max().item()
        worst = max(worst, err)
        print(f"chunk {ci}: max|d| = {err:.3e}")
    assert worst < TOL


def test_batched_windows_bit_identical_to_single_windows(full_codec):
    """`batch` windows of equal length in one call: every row equals its own single-window decode bit for bit (each
    window keeps its own causal left padding / attention window / RoPE positions)."""
    st = full_codec
    codes = torch.randint(0, 2048, (3, 33, 16), generator=torch.Generator().manual_seed(9)).cuda()
    both, _ = st.decode({"audio_codes": codes})
    for b in range(3):
        one, _ = st.decode({"audio_codes": codes[b:b + 1]})
        assert torch.equal(one[0], both[b]), b


def test_engine_decode_launches_no_library_kernel(full_codec):
    """Every kernel of a decode call comes from libfq3_engine.so (no cuDNN / cuBLAS / ATen kernel): names via the
    torch profiler (CUPTI); skipped when the profiler cannot trace CUDA here."""
    st = full_codec
    codes = torch.randint(0, 2048, (1, 33, 16), generator=torch.Generator().manual_seed(1)).cuda()
    st.decode({"audio_codes": codes})
    torch.cuda.synchronize()
    try:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            st.decode({"audio_codes": codes})
            torch.cuda.synchronize()
        names = [e.key for e in prof.key_averages() if getattr(e, "device_type", None) is not None and "Memcpy" not in e.key and "Memset" not in e.key]
    except Exception as ex:  # pragma: no cover
        pytest.skip(f"CUDA profiling unavailable: {ex!r}")
    kernels = [n for n in names if "kernel" in n or "(" in n]
    if not kernels:
        pytest.skip("profiler returned no kernel records")
    print(sorted(set(kernels)))
    foreign = [n for n in kernels if not any(s in n for s in ("fe::", "conv_gemm", "conv_out_kernel", "fq3", "cast_strided"))]
    assert not foreign, foreign


def _kernels_in_start_order(fn):
    """names of the kernels fn() launches, in start-time order (torch profiler, CUPTI); skips when CUDA cannot be traced"""
    torch.cuda.synchronize()
    try:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
              and not e.name.startswith(("Memcpy", "Memset"))]
    except Exception as ex:  # pragma: no cover
        pytest.skip(f"CUDA profiling unavailable: {ex!r}")
    if not ev:
        pytest.skip("profiler returned no kernel records")
    return [e.name for e in sorted(ev, key=lambda e: e.time_range.start)]


def _launch_geometry(st):
    """(launches of one decode, causal sites with history rows) of the codec geometry"""
    c = st.decoder.config
    L, U, nb = c.num_hidden_layers, len(c.upsampling_ratios), len(c.upsample_rates)
    # embedding mean; per pre-transformer layer 2 norms, 4 GEMMs, RoPE, attention; final norm; per upsampler
    # ConvTranspose GEMM, dwconv + LayerNorm, 2 GEMMs; conv_in; per decoder block ConvTranspose, 3 x (conv7, conv1); conv_out
    n_decode = 1 + 8 * L + 1 + 4 * U + 1 + 7 * nb + 1
    # sites with history: attention, dwconv, conv_in, per decoder block the ConvTranspose and the 3 conv7, conv_out
    return n_decode, L + U + 1 + 4 * nb + 1


def test_decode_launch_count_follows_the_codec_geometry(full_codec):
    """a decode of [2, 33, 16] makes the launches the codec geometry gives; push_streams on two fresh streams with the same
    codes makes those plus two history copies per causal site, and returns the same PCM"""
    st = full_codec
    n_decode, n_sites = _launch_geometry(st)
    assert (n_decode, n_sites) == (104, 28)
    codes = torch.randint(0, 2048, (2, 33, 16), generator=torch.Generator().manual_seed(41)).cuda()
    n0 = int(st._lib.fq3_codec_launch_count(st._h))
    one_shot, _ = st.decode({"audio_codes": codes})
    assert st.launches - n0 == n_decode
    streams = [st.open_stream() for _ in range(2)]
    n0 = st.launches
    streamed = st.push_streams(streams, codes)
    assert st.launches - n0 == n_decode + 2 * n_sites
    for a, b in zip(one_shot, streamed):
        assert torch.equal(a, b)
    for s in streams:
        s.close()


def test_one_shot_decode_is_the_stream_decode_without_history_copies(full_codec):
    """The one-shot decode and the stream decode run one codec forward: a decode of [2, 33, 16] launches the kernels of
    push_streams on two fresh streams with the same codes, in the same order, once the stream's history copies are
    removed."""
    st = full_codec
    n_decode, n_sites = _launch_geometry(st)
    codes = torch.randint(0, 2048, (2, 33, 16), generator=torch.Generator().manual_seed(42)).cuda()
    streams = [st.open_stream() for _ in range(2)]
    st.decode({"audio_codes": codes})
    st.push_streams(streams, codes)
    for s in streams:
        s.reset()
    one_shot = _kernels_in_start_order(lambda: st.decode({"audio_codes": codes}))
    streamed = _kernels_in_start_order(lambda: st.push_streams(streams, codes))
    copies = ("ext_build_kernel", "tail_save_kernel")
    assert len(one_shot) == n_decode and len(streamed) == n_decode + 2 * n_sites
    assert sum(any(k in n for k in copies) for n in streamed) == 2 * n_sites
    assert [n for n in streamed if not any(k in n for k in copies)] == one_shot
    for s in streams:
        s.close()


def test_push_streams_refuses_a_wrong_code_group_count_before_launching(full_codec):
    st = full_codec
    s = st.open_stream()
    n0 = int(st._lib.fq3_codec_launch_count(st._h))
    with pytest.raises(ValueError, match="16 code groups"):
        st.push_streams([s], torch.zeros(1, 4, 15, dtype=torch.long, device="cuda"))
    assert int(st._lib.fq3_codec_launch_count(st._h)) == n0 and s.frames == 0
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# stateful streaming codec (SURVEY 8(f) item 2): a stream's PCM equals the one-shot decode of the same codes
# ---------------------------------------------------------------------------------------------------------------------
def test_stateful_stream_equals_one_shot_decode(full_codec):
    """chunks of irregular sizes (incl. 1 frame and a chunk longer than the 72-frame attention window) pushed through one
    stream == fq3_codec_decode_codes of the whole sequence: every output row is the same arithmetic (causal model), so
    the bar is bit equality; the fp32 oracle bounds it at 1e-3 like every other codec path."""
    st = full_codec
    g = torch.Generator().manual_seed(21)
    sizes = [8, 8, 3, 1, 12, 80, 8]
    codes = torch.randint(0, 2048, (sum(sizes), 16), generator=g).cuda()
    whole, _ = st.decode({"audio_codes": codes[None]})
    stream = st.open_stream()
    got, pos = [], 0
    for n in sizes:
        got.append(stream.push(codes[pos:pos + n]))
        pos += n
        assert stream.frames == pos
    got = torch.cat(got)
    d = (got - whole[0]).abs().max().item()
    print(f"stream vs one-shot: max|d| = {d:.3e} over {got.numel()} samples")
    assert got.shape == whole[0].shape
    assert d == 0.0
    want = _oracle(st, codes)
    assert (got - want).abs().max().item() < TOL
    # reset -> the same stream object reproduces the beginning
    stream.reset()
    again = stream.push(codes[:8])
    assert torch.equal(again, got[: 8 * 1920])


def test_stateful_streams_batched_at_different_positions(full_codec):
    """three streams with different histories (fresh / 5 frames / 100 frames, the last one warmed without producing
    audio) advance 8 frames in ONE call; every row equals the tail of its own one-shot decode."""
    st = full_codec
    g = torch.Generator().manual_seed(22)
    hist = [0, 5, 100]
    seqs = [torch.randint(0, 2048, (h + 8, 16), generator=g).cuda() for h in hist]
    streams = [st.open_stream() for _ in hist]
    for s, q, h in zip(streams, seqs, hist):
        if h == 100:
            s.warm(q[:h])
        elif h:
            s.push(q[:h])
    out = st.push_streams(streams, torch.stack([q[-8:] for q in seqs]))
    for s, q, h, pcm in zip(streams, seqs, hist, out):
        whole, _ = st.decode({"audio_codes": q[None]})
        assert torch.equal(pcm, whole[0][h * 1920:]), h
        assert s.frames == h + 8


def test_stateful_window_policy_streams_the_non_streaming_audio(full_codec):
    """model-level: streaming_codec="stateful" through FasterQwen3TTS._stream_audio with an ICL reference of 174 frames:
    the concatenated chunks equal the non-streaming decode + reference trim (model.py:918-938) of the same codes."""
    import types
    from faster_qwen3_tts.model import FasterQwen3TTS
    st = full_codec
    g = torch.Generator().manual_seed(23)
    ref = torch.randint(0, 2048, (174, 16), generator=g).cuda()
    chunks = [torch.randint(0, 2048, (8, 16), generator=g).cuda() for _ in range(5)] + [torch.randint(0, 2048, (3, 16), generator=g).cuda()]
    owner = types.SimpleNamespace(streaming_codec="stateful", _to_numpy=FasterQwen3TTS._to_numpy)
    owner._make_window = types.MethodType(FasterQwen3TTS._make_window, owner)
    parts = [a for a, sr, _ in FasterQwen3TTS._stream_audio(owner, ((c, {}) for c in chunks), st, ref, 8, to_host=False)]
    assert [p.shape[0] for p in parts] == [c.shape[0] * 1920 for c in chunks]
    whole, _ = st.decode({"audio_codes": torch.cat([ref] + chunks)[None]})
    assert torch.equal(torch.cat(parts), whole[0][174 * 1920:])


def test_phase1_on_reference_stream_is_sample_identical_to_the_literal_window_policy(full_codec, monkeypatch):
    """The default window policy runs Phase 1 of an ICL request on a copy of the reference's warmed template stream instead
    of re-decoding [reference + everything so far] per chunk (model.py:1085-1112): every chunk must be bit-identical to the
    literal re-decode (FQ3_PHASE1_STREAM=0), Phase 2 included, for two requests sharing one cached reference."""
    from faster_qwen3_tts.model import _StreamWindow
    import types
    st = full_codec
    g = torch.Generator().manual_seed(31)
    ref = torch.randint(0, 2048, (174, 16), generator=g)          # host tensor, like the cached voice prompt holds it
    owner = types.SimpleNamespace(_to_numpy=None)
    st.clear_reference_cache()
    for req in range(2):
        chunks = [torch.randint(0, 2048, (8, 16), generator=g).cuda() for _ in range(6)] + [torch.randint(0, 2048, (5, 16), generator=g).cuda()]
        monkeypatch.setenv("FQ3_PHASE1_STREAM", "0")
        lit = _StreamWindow(owner, st, ref, 8, to_host=False)
        assert lit.p1 is None
        monkeypatch.setenv("FQ3_PHASE1_STREAM", "1")
        fast = _StreamWindow(owner, st, ref, 8, to_host=False)
        if req == 0:   # a voice never seen: first chunk literal, the template is warmed when the second chunk arrives
            assert fast.p1 is None and fast._p1_pending
        else:          # known voice: a copy of the warmed template is ready before the first chunk
            assert fast.p1 is not None and fast.p1.frames == 174
        for ci, c in enumerate(chunks):
            a, _ = lit.push(c)
            b, _ = fast.push(c)
            assert a.shape == b.shape == (c.shape[0] * 1920,), (req, ci)
            assert torch.equal(a, b), (req, ci)
            if ci == 1:
                assert fast.p1 is not None and fast.p1.frames == 174 + 16
        assert fast.p1 is None and fast.spf == lit.spf == 1920.0
    assert len(st._ref_templates) == 1        # one warmed template served both requests
