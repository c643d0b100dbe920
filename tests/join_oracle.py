"""numpy restatement of the join of a segmented request (faster_qwen3_tts/join.py, csrc/fq3_join.cu), written from the
rule alone: segments in order, 24 * pause_ms zeros between them, and at every inner boundary a raised-cosine fade over
F = 120 samples computed in float64 and applied as two float32 multiplications, fade-in first."""
import numpy as np

F = 120


def fade() -> np.ndarray:
    i = np.arange(F, dtype=np.float64)
    return (0.5 - 0.5 * np.cos(np.pi * (i + 0.5) / F)).astype(np.float32)


def join(segments, pause_ms: int) -> np.ndarray:
    w, S, out = fade(), len(segments), []
    for k, seg in enumerate(segments):
        x = np.asarray(seg, dtype=np.float32).copy()
        L = len(x)
        a = np.ones(L, np.float32)
        b = np.ones(L, np.float32)
        if k > 0:
            m = min(F, L)
            a[:m] = w[:m]
        if k < S - 1:
            m = min(F, L)
            b[L - m:] = w[:m][::-1]
        out.append((x * a) * b)
        if k < S - 1:
            out.append(np.zeros(24 * pause_ms, np.float32))
    return np.concatenate(out) if out else np.zeros(0, np.float32)
