"""numpy restatement of the join with a pause per boundary (``fq3_join_create_pauses``, ``join.Join(pauses=)``),
written from the rule alone: 24 * pauses_ms[0] zeros, seg_0, 24 * pauses_ms[1] zeros, ..., seg_{S-1},
24 * pauses_ms[S] zeros, with the raised-cosine fades of ``join_oracle.join`` at the inner boundaries only."""
import numpy as np

from join_oracle import F, fade


def join_pauses(segments, pauses_ms) -> np.ndarray:
    S = len(segments)
    assert len(pauses_ms) == S + 1
    w, out = fade(), [np.zeros(24 * pauses_ms[0], np.float32)]
    for k, seg in enumerate(segments):
        x = np.asarray(seg, dtype=np.float32).copy()
        L = len(x)
        a = np.ones(L, np.float32)
        b = np.ones(L, np.float32)
        m = min(F, L)
        if k > 0:
            a[:m] = w[:m]
        if k < S - 1:
            b[L - m:] = w[:m][::-1]
        out.append((x * a) * b)
        out.append(np.zeros(24 * pauses_ms[k + 1], np.float32))
    return np.concatenate(out)
