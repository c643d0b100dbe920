"""The weight tape's plan (csrc/fq3_tape.cuh) on the CPU: a small harness around tape_segments() and plan_tape(),
compiled with the engine's nvcc command, checks the plan's invariants for the model geometries in both layouts, the
planner's refusals, and pins the plan itself.  A planning mistake otherwise shows only as wrong numbers in a GPU parity
test, or as a producer waiting on a ring stage its consumers count differently."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "faster-qwen3-tts_b200", "csrc")
INCLUDE = os.path.join(ROOT, "include")

HARNESS = r"""
#include "@CSRC@/fq3_tape.cuh"
using namespace fq3;
static TapePlan plan;
static std::string err;
static std::vector<int32_t> segs;
// the plan of cfg on ncta CTAs: "" and its tables, or the refusal
extern "C" const char* tape_plan(const fq3_config* cfg, int ncta, int bf16, int64_t* info, const void** tabs) {
  const TapeSegments T = tape_segments(*cfg);
  err = plan_tape(T.segs, ncta, bf16 != 0, plan);
  segs.clear();
  for (const TapeSeg& s : T.segs) segs.insert(segs.end(), {s.rows, s.K, s.gu ? 1 : 0});
  const int64_t v[] = {(int64_t)plan.grps.size(), (int64_t)T.segs.size(), (int64_t)plan.pack.size(),
                       (int64_t)plan.tape_bytes, STAGE_BYTES, MAXGRP, T.seg_base[0], T.seg_head[0], T.seg_base[1],
                       T.seg_head[1], T.seg_mtp};
  for (int i = 0; i < 11; ++i) info[i] = v[i];
  tabs[0] = plan.grps.data(); tabs[1] = plan.segtab.data(); tabs[2] = plan.cta_grp_off.data();
  tabs[3] = plan.pack.data(); tabs[4] = segs.data();
  return err.c_str();
}
"""

GRP = np.dtype([("off16", "<u4"), ("row0", "<i4"), ("rows", "<u2"), ("m", "<u2"), ("ntiles", "<u2"), ("pad", "<u2")])
PACK = np.dtype([("tape_off", "<u8"), ("rowsrc_idx", "<u4"), ("rows", "<u2"), ("m", "<u2"), ("ntiles", "<u2"),
                 ("pad", "<u2"), ("K", "<i4")])
FULL, HALF, GU = 0, 1, 2

# (hidden, intermediate, layers, heads, kv heads, vocab) of talker and predictor, MTP projection
GEOMETRIES = {
    "1.7B": ((2048, 6144, 28, 16, 8, 3072), (1024, 3072, 5, 16, 8, 2048), True),
    "0.6B": ((1024, 3072, 28, 16, 8, 3072), (1024, 3072, 5, 16, 8, 2048), False),
    "tiny": ((512, 768, 3, 4, 2, 1280), (256, 512, 2, 4, 2, 256), True),
}

# sha256 of grps, segtab, cta_grp_off and the pack records (in tape order) at 132 CTAs, as the planner made them
# before it moved into fq3_tape.cuh.  A change of the tape's format or tile choice changes these on purpose.
PINNED = {
    ("1.7B", True): "26504617a3e308f40ca8f7c074a47c13040261b33c16c08ee7a9d8a4d2b4d8a4",
    ("1.7B", False): "fec990bee4e5c7f9f5619bc44468744630e1aeadb977d94229b03d7c780669fe",
    ("0.6B", True): "f3dabba6f12d2a09ed0835d955e938ea03a03dd4af99d823709bc7e535117f01",
    ("0.6B", False): "eb945e8dc3238feddc7056664993a20f3e16272e9b7e60afd6ecf6b303ac35a4",
    ("tiny", True): "d6ec7b1a7c57537682cf02015769cc80a2f9c62ce035e6316ebfe0bf815621db",
    ("tiny", False): "1ac747538ca045e3e9818a64b1a8fdd35b0658597174c0fd987a11ffe1f77975",
}


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    from faster_qwen3_tts.engine import Config
    d = tmp_path_factory.mktemp("tape")
    src, so = d / "tape_harness.cu", d / "tape_harness.so"
    src.write_text(HARNESS.replace("@CSRC@", CSRC))
    subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-shared",
                    "-Xcompiler", "-fPIC", "-I", INCLUDE, "-o", str(so), str(src)], check=True)
    lib = C.CDLL(str(so))
    lib.tape_plan.restype = C.c_char_p
    lib.tape_plan.argtypes = [C.POINTER(Config), C.c_int, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_void_p)]

    def plan(geom, ncta, bf16):
        t, p, mtp = geom
        cfg = Config(num_code_groups=16, has_mtp_projection=int(mtp))
        for st, g in ((cfg.talker, t), (cfg.predictor, p)):
            (st.hidden_size, st.intermediate_size, st.num_hidden_layers, st.num_attention_heads,
             st.num_key_value_heads, st.vocab_size) = g
        info, tabs = (C.c_int64 * 11)(), (C.c_void_p * 5)()
        err = lib.tape_plan(C.byref(cfg), ncta, int(bf16), info, tabs)
        if err:
            return err.decode()
        ngrp, nseg, npack, tape_bytes, stage, maxgrp = info[:6]

        def table(i, n, dtype):
            return np.frombuffer(C.string_at(tabs[i], n * np.dtype(dtype).itemsize), dtype=dtype).copy()
        return dict(grps=table(0, ngrp, GRP), segtab=table(1, ncta * nseg, "<u4").reshape(ncta, nseg),
                    cta_grp_off=table(2, ncta + 1, "<u4"), pack=table(3, npack, PACK),
                    segs=table(4, 3 * nseg, "<i4").reshape(nseg, 3), tape_bytes=tape_bytes, stage=stage,
                    maxgrp=maxgrp, seg_base=(info[6], info[8]), seg_head=(info[7], info[9]), seg_mtp=info[10])
    return plan


def expected_segments(geom):
    """(rows, K, gate/up) of every segment: per stack its layers' QKV, O, gate/up, down, then its heads (one talker head,
    15 predictor heads); the MTP projection last"""
    t, p, mtp = geom
    segs, base, head = [], [], []
    for (H, I, L, nh, nkv, V), nheads in ((t, 1), (p, 15)):
        qd, kd = nh * 128, nkv * 128
        base.append(len(segs))
        for _ in range(L):
            segs += [(qd + 2 * kd, H, 0), (H, qd, 0), (2 * I, H, 1), (H, I, 0)]
        head.append(len(segs))
        segs += [(V, H, 0)] * nheads
    seg_mtp = len(segs) if mtp else -1
    if mtp:
        segs.append((p[0], t[0], 0))
    return segs, tuple(base), tuple(head), seg_mtp


def digest(plan):
    h = hashlib.sha256()
    for name in ("grps", "segtab", "cta_grp_off", "pack"):
        h.update(plan[name].tobytes())
    return h.hexdigest()


def check_plan(plan, geom, ncta, bf16):
    segs, base, head, seg_mtp = expected_segments(geom)
    assert [tuple(s) for s in plan["segs"]] == segs
    assert (plan["seg_base"], plan["seg_head"], plan["seg_mtp"]) == (base, head, seg_mtp)
    grps, segtab, goff, pack = plan["grps"], plan["segtab"], plan["cta_grp_off"], plan["pack"]
    nseg = len(segs)
    # cta_grp_off: CTA c's groups are grps[goff[c]:goff[c + 1]], at most MAXGRP of them
    assert goff[0] == 0 and goff[-1] == len(grps) and np.all(np.diff(goff.astype(np.int64)) >= 0)
    assert np.diff(goff.astype(np.int64)).max() <= plan["maxgrp"]
    # per CTA, each segment's groups are contiguous, in segment order, and segtab points at them
    begin, count = segtab >> 8, segtab & 255
    assert np.all(begin == np.cumsum(count, axis=1) - count)
    assert np.all(count.sum(axis=1) == np.diff(goff.astype(np.int64)))
    seg_of = np.concatenate([np.repeat(np.arange(nseg), count[c]) for c in range(ncta)])
    rows_k = np.array(segs, dtype=np.int64)
    seg_k, seg_gu = rows_k[seg_of, 1], rows_k[seg_of, 2]
    row0, m, ntiles = grps["row0"].astype(np.int64), grps["m"].astype(np.int64), grps["ntiles"].astype(np.int64)
    if bf16:
        n_mt, kind = grps["rows"].astype(np.int64) & 0xFF, grps["rows"].astype(np.int64) >> 8
        assert np.all((kind == GU) == (seg_gu == 1)) and np.all(np.isin(n_mt[kind != HALF], (1, 2)))
        assert np.all(n_mt[kind == HALF] == 1)
        # rows covered: FULL 16 per m-tile, HALF 8, GU 8 gate/up pairs per m-tile (row0 counts pairs)
        start = np.where(kind == GU, 2 * row0, row0)
        length = np.select([kind == FULL, kind == HALF, kind == GU], [16 * n_mt, 8, 16 * n_mt])
        tile = n_mt * m * 2048
        assert np.all(m * ntiles * 64 == np.where(kind == HALF, seg_k // 2, seg_k))
    else:
        rows = grps["rows"].astype(np.int64)
        assert np.all(rows % 2 == 0) and np.all((rows > 0) & (rows <= 32))
        start, length, tile = row0, rows, rows * m * 512
        assert np.all(m * ntiles * 128 == seg_k)
    assert np.all(tile <= plan["stage"])
    # every row of every segment is covered by exactly one group of exactly one CTA
    order = np.lexsort((start, seg_of))
    s, st, ln = seg_of[order], start[order], length[order]
    for sg in range(nseg):
        a, b = st[s == sg], ln[s == sg]
        assert a[0] == 0 and np.all(a[1:] == a[:-1] + b[:-1]) and a[-1] + b[-1] == segs[sg][0], sg
    # offsets advance by each group's bytes in consumption order; each CTA's slice starts 1024-aligned
    off = 0
    nbytes = tile * ntiles
    for c in range(ncta):
        g0, g1 = goff[c], goff[c + 1]
        want = off + np.concatenate([[0], np.cumsum(nbytes[g0:g1])[:-1]])
        assert np.all(grps["off16"][g0:g1].astype(np.int64) * 16 == want), c
        off = -(-(off + nbytes[g0:g1].sum()) // 1024) * 1024
    assert off == plan["tape_bytes"]
    # one pack record per group, in tape order, reading the group's rows of the row-source table
    rowsrc0 = np.concatenate([[0], np.cumsum(rows_k[:, 0])])
    assert len(pack) == len(grps)
    assert np.all(pack["tape_off"] == grps["off16"].astype(np.uint64) * 16)
    for f in ("rows", "m", "ntiles"):
        assert np.all(pack[f] == grps[f])
    assert np.all(pack["K"] == seg_k)
    assert np.all(pack["rowsrc_idx"] == rowsrc0[seg_of] + start)


@pytest.mark.parametrize("ncta", [132, 114])
@pytest.mark.parametrize("bf16", [True, False], ids=["bf16", "fp32"])
@pytest.mark.parametrize("size", list(GEOMETRIES))
def test_plan_invariants(harness, size, bf16, ncta):
    plan = harness(GEOMETRIES[size], ncta, bf16)
    assert isinstance(plan, dict), plan
    check_plan(plan, GEOMETRIES[size], ncta, bf16)


@pytest.mark.parametrize("bf16", [True, False], ids=["bf16", "fp32"])
def test_plan_tiny_on_few_ctas(harness, bf16):
    plan = harness(GEOMETRIES["tiny"], 7, bf16)
    assert isinstance(plan, dict), plan
    check_plan(plan, GEOMETRIES["tiny"], 7, bf16)


@pytest.mark.parametrize("bf16", [True, False], ids=["bf16", "fp32"])
@pytest.mark.parametrize("size", list(GEOMETRIES))
def test_plan_is_pinned(harness, size, bf16):
    assert digest(harness(GEOMETRIES[size], 132, bf16)) == PINNED[(size, bf16)]


def test_plan_refusals(harness):
    (H, I, L, nh, nkv, V), p, mtp = GEOMETRIES["tiny"]
    assert harness(((576, I, L, nh, nkv, V), p, mtp), 132, True) == \
        "segment 0: rows 1024 / K 576 not tileable for the bf16 tensor-core tape"
    assert harness(((H, I, L, nh, nkv, 1279), p, mtp), 132, False) == \
        "segment 12: rows 1279 must be even and K 512 a multiple of 128"
    assert harness(GEOMETRIES["1.7B"], 7, True) == "CTA 0 has 3027 row groups (> 512)"
