// fq3_decode_batch.cuh -- batched persistent decode kernel (sm_90a): up to 32 request slots share ONE pass over the
// weight tape per step (BASELINE config 4: concurrent requests per GPU; the reference's batch handling is the
// left-padded prompt batch of faster_qwen3_tts/model.py:774-787 with per-row pad counts, talker_graph.py:177-187).
//
// Same tape, same producer warp / TMA ring, same grid barrier and the same per-element arithmetic (rounding points,
// accumulation order inside a warp, cross-warp summation order) as the single-sequence kernel in fq3_decode.cuh: row b
// of a batched launch produces bit-for-bit the codes a single-sequence launch produces for that request (tested).  The
// attention functions, the fp32 GEMV, the talker's draw arguments, the step advance, the state record and the
// producer's frame walk are the single-sequence kernel's own, called with this slot's pointers.
//
// What changes with B > 1:
//   * activations live in global memory (L2-resident) as [column][K] matrices, column = slot (predictor pass 0: column
//     = token * B + slot).  Every GEMV becomes a skinny GEMM: the activation matrix is the mma.m16n8k16 B operand, read
//     straight from L2 in fragment order (the tape's bf16 column permutation makes a lane's 32 bytes contiguous), up to
//     four n-groups of 8 columns per pass over a ring tile; more than 32 columns (fp32 parity mode: more than 8) replay
//     the segment (the CTA's slice is L2-resident by then).
//   * cheap per-row work that the single-sequence kernel computes redundantly in every CTA is distributed: CTA c
//     serves slot c % B (RMSNorm rows, predictor attention, sampling); talker attention items (slot, q-head) are dealt
//     round-robin to all CTAs.  Results that other CTAs need go through global memory + the grid barrier.
//   * every slot carries its own position, left-pad count, rope delta, trailing-text stream, sampling parameters,
//     uniforms, penalty bitmap and KV caches (SlotParams); slots finish independently (EOS / max_new / max_seq_len).
#pragma once
#include "fq3_decode.cuh"

namespace fq3 {

constexpr int MAXB = 32;          // slots per launch
constexpr int MAXCOL = 2 * MAXB;  // activation columns (predictor pass 0 carries 2 tokens per slot)

// phase accounting (dbg_on & 2): CTA 0 / thread 0 charges the clock64 cycles since the last mark to the category that
// was current; dumped to the debug buffer at the end of the launch (tools/batch_bench.py --phases)
enum { PC_OTHER = 0, PC_GEMV = 1, PC_BARRIER = 2, PC_NORM = 3, PC_ATTN = 4, PC_SAMPLE = 5, PC_N = 6 };
__device__ __forceinline__ void pmark(Ctx& c, int cat) {
  if ((c.P.dbg_on & 2) && blockIdx.x == 0 && c.tid == 0) {
    Smem& s = SMEM();
    const long long now = clock64();
    s.prof[2 + (int)s.prof[1]] += now - s.prof[0];
    s.prof[0] = now;
    s.prof[1] = cat;
  }
}
__device__ __forceinline__ void grid_sync_p(Ctx& c, int next_cat) {
  pmark(c, PC_BARRIER);
  grid_sync(c);
  pmark(c, next_cat);
}

// ------------------------------------------------------------------------------------------------------------
// GEMV epilogues (what the single-sequence kernel expresses as lambdas)
// ------------------------------------------------------------------------------------------------------------
enum EpiKind { EP_F32 = 0, EP_RESID = 1, EP_SWIGLU = 2, EP_BIAS = 3 };
struct EpiB {
  int kind;
  float* outf;        // fp32 destination [col][ldo]            (F32 / RESID / BIAS)
  void* outd;         // model-dtype destination [col][ldo]     (SWIGLU)
  int ldo;
  const float* res;   // RESID: residual [col][ldres]
  int ldres;
  const void* bias;   // BIAS: [rows] model dtype or nullptr
};
template <bool BF>
__device__ __forceinline__ float epi_pre(const EpiB& e, int row, int col) {
  if (e.kind == EP_RESID) return __ldcg(e.res + (size_t)col * e.ldres + row);
  if (e.kind == EP_BIAS) return e.bias ? ldw<BF>(e.bias, row) : 0.f;
  return 0.f;
}
template <bool BF>
__device__ __forceinline__ void epi_apply(const EpiB& e, int row, int col, float v, float vup, float aux) {
  if (e.kind == EP_F32) {
    e.outf[(size_t)col * e.ldo + row] = rnd<BF>(v);
  } else if (e.kind == EP_RESID) {
    e.outf[(size_t)col * e.ldo + row] = rnd<BF>(aux + rnd<BF>(v));
  } else if (e.kind == EP_SWIGLU) {
    const float gte = rnd<BF>(v), up = rnd<BF>(vup);
    const float sl = rnd<BF>(gte / (1.0f + expf(-gte)));
    stw<BF>(e.outd, (size_t)col * e.ldo + row, rnd<BF>(sl * up));
  } else {
    e.outf[(size_t)col * e.ldo + row] = rnd<BF>(v + aux);
  }
}

// ------------------------------------------------------------------------------------------------------------
// bf16 tensor-core GEMV over up to 8*NG activation columns (one pass over the segment's ring tiles).
// xg: bf16 [col][ldx] in global memory; columns col0 .. col0+ncols.  Per-column arithmetic identical to gemv_mma.
// ------------------------------------------------------------------------------------------------------------
template <int NG>
__device__ __noinline__ void gemv_mma_b(Ctx& c, int seg, int K, const __nv_bfloat16* __restrict__ xg, int ldx, int col0,
                                        int ncols, const EpiB e) {
  constexpr int NACC = 2 * NG;
  float* red = SMEM().xs;  // [NCW][NACC][4][32] partial accumulators (spills over into xin for NG = 4)
  const uint32_t st = SMEM().seg[seg];
  const int gbeg = seg_begin(st), gn = seg_count(st);
  const int gq = c.lane >> 2, t = c.lane & 3;
  const int ngr = (ncols + 7) >> 3;   // n-groups in use (FULL / GU tiles)
  const int ngh = (ncols + 3) >> 2;   // token groups of 4 (HALF tiles)
  for (int gi = 0; gi < gn; ++gi) {
    const Grp g = SMEM().grp[gbeg + gi];
    const int n_mt = grp_nmt(g.rows), kind = grp_kind(g.rows), G = g.m;
    const int nacc = kind == 1 ? ngh : n_mt * NG;
    float aux[4] = {0.f, 0.f, 0.f, 0.f};
    if (c.warp < nacc) {
      if (kind == 0) {
        const int mt = c.warp / NG, ng = c.warp % NG;
        const int rA = g.row0 + mt * 16 + gq, cA = ng * 8 + 2 * t;
        if (cA < ncols) { aux[0] = epi_pre<true>(e, rA, col0 + cA); aux[2] = epi_pre<true>(e, rA + 8, col0 + cA); }
        if (cA + 1 < ncols) { aux[1] = epi_pre<true>(e, rA, col0 + cA + 1); aux[3] = epi_pre<true>(e, rA + 8, col0 + cA + 1); }
      } else if (kind == 1) {
        const int tok = c.warp * 4 + t;
        if (tok < ncols) aux[0] = epi_pre<true>(e, g.row0 + gq, col0 + tok);
      }
    }
    // per-lane B-operand row pointers
    const __nv_bfloat16* xb[NACC];
    if (kind != 1) {
#pragma unroll
      for (int ng = 0; ng < NG; ++ng) {
        const int col = ng * 8 + gq;
        xb[ng] = xg + (size_t)(col0 + (col < ncols ? col : 0)) * ldx + 16 * t;
      }
#pragma unroll
      for (int ng = NG; ng < NACC; ++ng) xb[ng] = xb[0];
    } else {
#pragma unroll
      for (int a = 0; a < NACC; ++a) {
        const int tok = a * 4 + (gq >> 1);
        xb[a] = xg + (size_t)(col0 + (tok < ncols ? tok : 0)) * ldx + (gq & 1) * (K >> 1) + 16 * t;
      }
    }
    float acc[NACC][4];
#pragma unroll
    for (int a = 0; a < NACC; ++a)
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[a][r] = 0.f;
    for (int tl = 0; tl < g.ntiles; ++tl) {
      const int stage = (int)(c.tile_ctr % NS);
      const uint32_t par = (c.tile_ctr / NS) & 1u;
      mbar_wait(&SMEM().full[stage], par);
      const uint8_t* tile = SMEM().ring[stage];
      for (int qq = c.warp; qq < G; qq += NCW) {
        const int kg = tl * G + qq;
        if (kind != 1) {
          uint4 blo[NG], bhi[NG];
#pragma unroll
          for (int ng = 0; ng < NG; ++ng) {
            blo[ng] = __ldcg(reinterpret_cast<const uint4*>(xb[ng] + 64 * kg));
            bhi[ng] = __ldcg(reinterpret_cast<const uint4*>(xb[ng] + 64 * kg + 8));
          }
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            if (mt < n_mt) {
              const uint4* A = reinterpret_cast<const uint4*>(tile + ((size_t)(mt * G + qq) * 4) * 512) + c.lane;
              const uint4 a0 = A[0], a1 = A[32], a2 = A[64], a3 = A[96];
#pragma unroll
              for (int ng = 0; ng < NG; ++ng) {
                if (ng < ngr) {
                  mma_bf16(acc[mt * NG + ng], a0, blo[ng].x, blo[ng].y);
                  mma_bf16(acc[mt * NG + ng], a1, blo[ng].z, blo[ng].w);
                  mma_bf16(acc[mt * NG + ng], a2, bhi[ng].x, bhi[ng].y);
                  mma_bf16(acc[mt * NG + ng], a3, bhi[ng].z, bhi[ng].w);
                }
              }
            }
          }
        } else {
          const uint4* A = reinterpret_cast<const uint4*>(tile + ((size_t)qq * 4) * 512) + c.lane;
          const uint4 a0 = A[0], a1 = A[32], a2 = A[64], a3 = A[96];
#pragma unroll
          for (int a = 0; a < NACC; ++a) {
            if (a < ngh) {
              const uint4 blo = __ldcg(reinterpret_cast<const uint4*>(xb[a] + 64 * kg));
              const uint4 bhi = __ldcg(reinterpret_cast<const uint4*>(xb[a] + 64 * kg + 8));
              mma_bf16(acc[a], a0, blo.x, blo.y);
              mma_bf16(acc[a], a1, blo.z, blo.w);
              mma_bf16(acc[a], a2, bhi.x, bhi.y);
              mma_bf16(acc[a], a3, bhi.z, bhi.w);
            }
          }
        }
      }
      __syncwarp();
      if (c.lane == 0) mbar_arrive(&SMEM().empty[stage]);
      c.tile_ctr++;
    }
#pragma unroll
    for (int a = 0; a < NACC; ++a)
      if (a < nacc)
#pragma unroll
        for (int r = 0; r < 4; ++r) red[((c.warp * NACC + a) * 4 + r) * 32 + c.lane] = acc[a][r];
    csync();
    if (c.warp < nacc) {
      const int a = c.warp;
      float cv[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        float sm = 0.f;
#pragma unroll
        for (int w = 0; w < NCW; ++w) sm += red[((w * NACC + a) * 4 + r) * 32 + c.lane];
        cv[r] = sm;
      }
      if (kind == 1) {
        const int tok = a * 4 + t;
        if (tok < ncols) epi_apply<true>(e, g.row0 + gq, col0 + tok, cv[0] + cv[3], 0.f, aux[0]);
      } else {
        const int mt = a / NG, ng = a % NG;
        const int cA = ng * 8 + 2 * t;
        if (kind == 2) {
          const int pair = g.row0 + mt * 8 + gq;
          if (cA < ncols) epi_apply<true>(e, pair, col0 + cA, cv[0], cv[2], 0.f);
          if (cA + 1 < ncols) epi_apply<true>(e, pair, col0 + cA + 1, cv[1], cv[3], 0.f);
        } else {
          const int rA = g.row0 + mt * 16 + gq;
          if (cA < ncols) { epi_apply<true>(e, rA, col0 + cA, cv[0], 0.f, aux[0]); epi_apply<true>(e, rA + 8, col0 + cA, cv[2], 0.f, aux[2]); }
          if (cA + 1 < ncols) { epi_apply<true>(e, rA, col0 + cA + 1, cv[1], 0.f, aux[1]); epi_apply<true>(e, rA + 8, col0 + cA + 1, cv[3], 0.f, aux[3]); }
        }
      }
    }
    csync();
  }
}

// ------------------------------------------------------------------------------------------------------------
// fp32 (parity mode) GEMV over up to 8 activation columns of a global [col][ldx] matrix: gemv_seg with the EpiB
// epilogue.
// ------------------------------------------------------------------------------------------------------------
__device__ __noinline__ void gemv_seg_b(Ctx& c, int seg, const float* __restrict__ xg, int ldx, int col0, int ncols,
                                        const EpiB e) {
  constexpr int NT = 8;
  gemv_seg<NT, true>(c, seg, xg + (size_t)col0 * ldx, ldx, ncols, [&](int row0, const float* v0, const float* v1) {
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      if (t < ncols) {
        if (e.kind == EP_SWIGLU) {
          epi_apply<false>(e, row0 >> 1, col0 + t, v0[t], v1[t], 0.f);
        } else {
          epi_apply<false>(e, row0, col0 + t, v0[t], 0.f, epi_pre<false>(e, row0, col0 + t));
          epi_apply<false>(e, row0 + 1, col0 + t, v1[t], 0.f, epi_pre<false>(e, row0 + 1, col0 + t));
        }
      }
    }
  });
}

// column blocks per segment pass: the producer replays the segment once per block
__host__ __device__ __forceinline__ int col_blocks(bool bf, int ncols) { return bf ? (ncols + 31) / 32 : (ncols + 7) / 8; }

template <bool BF>
__device__ __forceinline__ void gemv_b(Ctx& c, int seg, int K, const void* xg, int ldx, int ncols, const EpiB& e) {
  if constexpr (BF) {
    const __nv_bfloat16* x = reinterpret_cast<const __nv_bfloat16*>(xg);
    for (int c0 = 0; c0 < ncols; c0 += 32) {
      const int n = min(32, ncols - c0);
      if (n <= 8) gemv_mma_b<1>(c, seg, K, x, ldx, c0, n, e);
      else if (n <= 16) gemv_mma_b<2>(c, seg, K, x, ldx, c0, n, e);
      else gemv_mma_b<4>(c, seg, K, x, ldx, c0, n, e);
    }
  } else {
    const float* x = reinterpret_cast<const float*>(xg);
    for (int c0 = 0; c0 < ncols; c0 += 8) gemv_seg_b(c, seg, x, ldx, c0, min(8, ncols - c0), e);
  }
}

// ------------------------------------------------------------------------------------------------------------
// RMSNorm of one activation row (values from `prov`) into a model-dtype row of the GEMV input matrix.  Arithmetic and
// summation order of norm_stage(); the writes of a row are shared by `nparts` CTAs (every one of them forms the full
// sum of squares).  xcopy / hcopy: optional fp32 copies of the raw row (residual stream) / of the normalised row.
// ------------------------------------------------------------------------------------------------------------
template <bool BF, class Prov>
__device__ __forceinline__ void norm_row_b(Ctx& c, Prov prov, const void* w, size_t woff, int H, float eps, void* xn,
                                           float* xcopy, float* hcopy, int part, int nparts) {
  float v[NORM_E], wv[NORM_E];
#pragma unroll
  for (int i = 0; i < NORM_E; ++i) {
    const int k = c.tid + i * NCT;
    v[i] = 0.f;
    wv[i] = 0.f;
    if (k < H) {
      v[i] = prov(k);
      wv[i] = ldw<BF>(w, woff + k);
    }
  }
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < NORM_E; ++i) ss += v[i] * v[i];
  ss = block_sum(c, ss);
  const float r = 1.0f / sqrtf(ss / (float)H + eps);
#pragma unroll
  for (int i = 0; i < NORM_E; ++i) {
    const int k = c.tid + i * NCT;
    if (k < H && (i % nparts) == part) {
      const float y = rnd<BF>(wv[i] * rnd<BF>(v[i] * r));
      stw<BF>(xn, k, y);
      if (xcopy) xcopy[k] = v[i];
      if (hcopy) hcopy[k] = y;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// per-CTA view of a batched launch
// ------------------------------------------------------------------------------------------------------------
struct BView {
  int B;       // columns (slots) of this launch
  int b;       // the slot this CTA serves (cta % B)
  int rank;    // rank of this CTA among the CTAs serving slot b
  int gsz;     // CTAs serving slot b
};

// One pass through a transformer stack for nt tokens per slot (columns t*B + b).  On entry the layer-0 input norm has
// been written (XNB) together with the raw rows (XB) -- both published by the barrier this function starts with.  On
// return XNB rows [0,B) hold the final-norm hidden of the last token of every running slot (published), hcopy: the
// talker's past_hidden copy.
template <bool BF, bool TALKER>
__device__ void stack_b(Ctx& c, const StackDev& S, const BView& v, int nt, uint32_t run, int pass_slot0) {
  const KParams& P = c.P;
  const int B = v.B, ncols = nt * B;
  const bool mine = (run >> v.b) & 1u;
  const int nparts = min(v.gsz, S.H / NCT);
  const SlotParams& me = P.sl[v.b];
  for (int l = 0; l < S.L; ++l) {
    if (l > 0) {
      if (mine && v.rank < nparts)
        for (int t = 0; t < nt; ++t) {
          const int col = t * B + v.b;
          const float* src = P.XB + (size_t)col * P.ldX;
          norm_row_b<BF>(c, [&](int k) { return __ldcg(src + k); }, S.ln_in, (size_t)l * S.H, S.H, S.eps,
                         reinterpret_cast<uint8_t*>(P.XNB) + (size_t)col * P.ldX * (BF ? 2 : 4), nullptr, nullptr, v.rank, nparts);
        }
    }
    grid_sync_p(c, PC_GEMV);
    // ---- QKV rows
    {
      EpiB e{EP_F32, P.QKVB, nullptr, P.ldQKV, nullptr, 0, nullptr};
      gemv_b<BF>(c, S.seg_base + 4 * l + 0, S.H, P.XNB, P.ldX, ncols, e);
    }
    grid_sync_p(c, PC_ATTN);
    // ---- attention
    if constexpr (TALKER) {
      // items (running slot, q-head) dealt round-robin to the CTAs
      const int nrun = SMEM().runl[32];
      for (int idx = blockIdx.x; idx < nrun * S.nH; idx += gridDim.x) {
        const int b = SMEM().runl[idx / S.nH], h = idx % S.nH;
        const SlotParams& sp = P.sl[b];
        const int pos = sp.prefill_len + SMEM().bst[ST_STEP][b];
        // the column's page table into shared memory for the item's key loops (the previous item's last barrier
        // freed it; this one publishes it)
        for (int i = c.tid; i < (P.max_seq_len + KV_PAGE - 1) / KV_PAGE; i += NCT) SMEM().kvtab[i] = sp.kv_pages[i];
        csync();
        attention_head<BF>(c, S, l, h, P.QKVB + (size_t)b * P.ldQKV, sp.kv, SMEM().kvtab,
                           reinterpret_cast<uint8_t*>(P.ATTB) + (size_t)b * P.ldATT * (BF ? 2 : 4), pos,
                           pos + sp.rope_delta, sp.n_left_pad);
      }
    } else {
      if (mine && v.rank == 0) {
        const float* q0 = P.QKVB + (size_t)v.b * P.ldQKV;
        uint8_t* a0 = reinterpret_cast<uint8_t*>(P.ATTB) + (size_t)v.b * P.ldATT * (BF ? 2 : 4);
        auto to_att = [&](int t, int i, float x) { stw<BF>(a0, (size_t)t * B * P.ldATT + i, x); };
        if (nt == 1) attention_small_all<BF, 1>(c, S, l, pass_slot0, pass_slot0, q0, 0, me.pkc, me.pvc, true, nullptr, to_att);
        else attention_small_all<BF, 2>(c, S, l, 0, 0, q0, (size_t)B * P.ldQKV, me.pkc, me.pvc, true, nullptr, to_att);
      }
    }
    grid_sync_p(c, PC_GEMV);
    // ---- o_proj + residual
    {
      EpiB e{EP_RESID, P.X1B, nullptr, P.ldX, P.XB, P.ldX, nullptr};
      gemv_b<BF>(c, S.seg_base + 4 * l + 1, S.qd, P.ATTB, P.ldATT, ncols, e);
    }
    grid_sync_p(c, PC_NORM);
    // ---- post-attention norm
    if (mine && v.rank < nparts)
      for (int t = 0; t < nt; ++t) {
        const int col = t * B + v.b;
        const float* src = P.X1B + (size_t)col * P.ldX;
        norm_row_b<BF>(c, [&](int k) { return __ldcg(src + k); }, S.ln_post, (size_t)l * S.H, S.H, S.eps,
                       reinterpret_cast<uint8_t*>(P.XNB) + (size_t)col * P.ldX * (BF ? 2 : 4), nullptr, nullptr, v.rank, nparts);
      }
    grid_sync_p(c, PC_GEMV);
    // ---- gate/up + SiLU*up
    {
      EpiB e{EP_SWIGLU, nullptr, P.ACTB, P.ldACT, nullptr, 0, nullptr};
      gemv_b<BF>(c, S.seg_base + 4 * l + 2, S.H, P.XNB, P.ldX, ncols, e);
    }
    grid_sync_p(c, PC_GEMV);
    // ---- down + residual
    {
      EpiB e{EP_RESID, P.XB, nullptr, P.ldX, P.X1B, P.ldX, nullptr};
      gemv_b<BF>(c, S.seg_base + 4 * l + 3, S.I, P.ACTB, P.ldACT, ncols, e);
    }
    grid_sync_p(c, PC_NORM);
  }
  // final norm of the last token -> XNB row b (head GEMV input); talker: also the slot's past_hidden
  if (mine && v.rank < nparts) {
    const int col = (nt - 1) * B + v.b;
    const float* src = P.XB + (size_t)col * P.ldX;
    norm_row_b<BF>(c, [&](int k) { return __ldcg(src + k); }, S.ln_f, 0, S.H, S.eps,
                   reinterpret_cast<uint8_t*>(P.XNB) + (size_t)v.b * P.ldX * (BF ? 2 : 4), nullptr,
                   TALKER ? me.past_hidden : nullptr, v.rank, nparts);
  }
  grid_sync_p(c, PC_GEMV);
}

// ------------------------------------------------------------------------------------------------------------
// producer warp of the batched kernel: producer_main()'s frame walk, every segment replayed once per column block
// (see gemv_b); the talker's attention is never split
// ------------------------------------------------------------------------------------------------------------
template <bool BF>
__device__ __noinline__ void producer_batch_main(const KParams& P) {
  const int lane = (int)(threadIdx.x & 31u);
  if (lane == 0) {
    Producer<BF> pr(P);
    if (P.mode == MODE_GEMV_TEST) pr.seg(P.gt_seg, col_blocks(BF, P.gt_ncols));
    else
      for (int f = 0; f < P.n_frames && !pr.stopped; ++f)
        pr.frame(col_blocks(BF, 2 * P.nslots), col_blocks(BF, P.nslots), -1, 0);
    pr.finish();
  }
}

// ------------------------------------------------------------------------------------------------------------
// the batched kernel: generate.py:149-199 / streaming.py:106-173 for every slot of the launch, lock-step per frame
// ------------------------------------------------------------------------------------------------------------
template <bool BF>
__global__ void __launch_bounds__(NTHREADS, 1) fq3_decode_batch_kernel(const __grid_constant__ KParams P) {
  Smem& s = SMEM();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cta = blockIdx.x;
  const int B = P.nslots;
  BView v;
  v.B = B;
  v.b = cta % B;
  v.rank = cta / B;
  v.gsz = ((int)gridDim.x - v.b + B - 1) / B;
  const SlotParams& me = P.sl[v.b];
  cta_prologue(P, P.mode == MODE_GEMV_TEST ? nullptr : me.seen);
  if (tid < B && P.mode != MODE_GEMV_TEST) {
    const int* st = P.sl[tid].state;
    s.bst[ST_TOKEN][tid] = st[ST_TOKEN]; s.bst[ST_STEP][tid] = st[ST_STEP]; s.bst[ST_GEN][tid] = st[ST_GEN];
    s.bst[ST_FIN][tid] = FQ3_RUNNING; s.bst[ST_EMIT][tid] = 0;
  }
  __syncthreads();

  if (warp == NCW) {
    producer_batch_main<BF>(P);
  } else {
    Ctx c{P, tid, warp, lane, 0u, 0u};
    const int Ht = P.t.H;
    const size_t esz = BF ? 2 : 4;
    const StackDev& Sp = P.p;
    if (tid == 0) {
      for (int i = 0; i < 12; ++i) s.prof[i] = 0;
      s.prof[0] = clock64();
    }
    const int npp = min(v.gsz, Sp.H / NCT);   // CTAs sharing the writes of a predictor norm row
    const int npt = min(v.gsz, Ht / NCT);     // ... of a talker norm row
    if (P.mode == MODE_GEMV_TEST) {
      EpiB e{P.gt_swiglu ? EP_SWIGLU : EP_F32, reinterpret_cast<float*>(P.gt_out), P.gt_out,
             P.gt_swiglu ? P.gt_rows / 2 : P.gt_rows, nullptr, 0, nullptr};
      gemv_b<BF>(c, P.gt_seg, P.gt_K, P.gt_x, P.gt_K, P.gt_ncols, e);
      grid_sync(c);
    }
    while (P.mode != MODE_GEMV_TEST) {
      // ---- which slots run this frame (identical decision in every CTA)
      if (warp == 0) {
        bool r = false;
        if (lane < B && s.bst[ST_FIN][lane] == FQ3_RUNNING && s.bst[ST_EMIT][lane] < P.sl[lane].n_frames) {   // own budget
          if (s.bst[ST_STEP][lane] >= P.sl[lane].max_new) s.bst[ST_FIN][lane] = FQ3_FIN_MAX_NEW;
          else if (s.bst[ST_TOKEN][lane] == P.eos) s.bst[ST_FIN][lane] = FQ3_FIN_EOS;
          else r = !(P.sl[lane].text_open && s.bst[ST_GEN][lane] >= P.sl[lane].trailing_len);   // open text: wait for the row
        }
        const unsigned m = __ballot_sync(0xffffffffu, r);
        if (lane == 0) s.ibc[0] = (int)m;
      }
      csync();
      const uint32_t run = (uint32_t)s.ibc[0];
      csync();
      if (run == 0u) break;
      const bool mine = (run >> v.b) & 1u;
      const int token = s.bst[ST_TOKEN][v.b], step = s.bst[ST_STEP][v.b], gen_step = s.bst[ST_GEN][v.b];
      const float* urow = me.uniforms ? me.uniforms + (size_t)(step + 1) * 16 : nullptr;
      if (mine && tid == 0) {
        s.codes[0] = token;
        s.seen[token >> 5] |= 1u << (token & 31);
      }
      csync();
      // ================= predictor: 15 passes (predictor_graph.py:115-167) =================
      if (P.has_mtp) {
        // pass-0 input rows -> PINB (model dtype): column b = past_hidden, column B + b = codec_embedding(token)
        if (mine && v.rank < 2) {
          for (int t = 0; t < 2; ++t) {
            if (v.gsz >= 2 && t != v.rank) continue;
            uint8_t* dst = reinterpret_cast<uint8_t*>(P.PINB) + (size_t)(t * B + v.b) * HMAX * esz;
            for (int k = tid; k < Ht; k += NCT)
              stw<BF>(dst, k, t == 0 ? __ldcg(me.past_hidden + k) : ldw<BF>(P.t_embed, (size_t)token * Ht + k));
          }
        }
        grid_sync_p(c, PC_GEMV);
        EpiB e{EP_BIAS, P.XB, nullptr, P.ldX, nullptr, 0, P.mtp_b};
        gemv_b<BF>(c, P.seg_mtp, Ht, P.PINB, HMAX, 2 * B, e);
        grid_sync_p(c, PC_NORM);
      }
      for (int i = 0; i < P.ncb; ++i) {
        const int nt = (i == 0) ? 2 : 1;
        // ---- layer-0 input norm of this pass (raw rows -> XB, normalised rows -> XNB)
        pmark(c, PC_NORM);
        if (mine && v.rank < npp) {
          for (int t = 0; t < nt; ++t) {
            const int col = t * B + v.b;
            uint8_t* xn = reinterpret_cast<uint8_t*>(P.XNB) + (size_t)col * P.ldX * esz;
            float* xr = P.XB + (size_t)col * P.ldX;
            if (i == 0 && P.has_mtp) {
              norm_row_b<BF>(c, [&](int k) { return __ldcg(xr + k); }, Sp.ln_in, 0, Sp.H, Sp.eps, xn, nullptr, nullptr, v.rank, npp);
            } else if (i == 0) {
              norm_row_b<BF>(c, [&](int k) { return t == 0 ? __ldcg(me.past_hidden + k) : ldw<BF>(P.t_embed, (size_t)token * Ht + k); },
                             Sp.ln_in, 0, Sp.H, Sp.eps, xn, xr, nullptr, v.rank, npp);
            } else {
              const int prev = s.codes[i];  // code sampled by pass i-1
              const void* tab = P.has_mtp ? P.mtp_tab : P.p_embeds;
              const size_t off = ((size_t)(i - 1) * Sp.V + prev) * (P.has_mtp ? Sp.H : Ht);
              norm_row_b<BF>(c, [&](int k) { return ldw<BF>(tab, off + k); }, Sp.ln_in, 0, Sp.H, Sp.eps, xn, xr, nullptr, v.rank, npp);
            }
          }
        }
        const int slot0 = (i == 0) ? 0 : i + 1;
        stack_b<BF, false>(c, Sp, v, nt, run, slot0);
        {
          EpiB e{EP_F32, P.LOGB, nullptr, VMAX, nullptr, 0, nullptr};
          gemv_b<BF>(c, Sp.seg_head + i, Sp.H, P.XNB, P.ldX, B, e);
        }
        grid_sync_p(c, PC_SAMPLE);
        if (mine) {
          SampleArgs sa;
          sa.logits = P.LOGB + (size_t)v.b * VMAX; sa.V = Sp.V; sa.sp = me.sp_p;
          sa.u = (me.sp_p.do_sample && urow) ? __ldg(urow + 1 + i) : 0.f;
          sa.use_penalty = false; sa.sup0 = Sp.V; sa.suppress_eos = false; sa.eos = -1;
          // the slot's rank-0 CTA writes the log-probabilities, as it writes the codes
          if (me.logprob_out && v.rank == 0) sa.lp = me.logprob_out + (size_t)s.bst[ST_EMIT][v.b] * 16 + 1 + i;
          const int tok = sample_block<BF>(c, sa);
          if (tid == 0) s.codes[i + 1] = tok;
          csync();
        }
      }
      pmark(c, PC_OTHER);
      // ---- emit the frame (generate.py:159): cat(cb0, 15 ids)
      if (mine && v.rank == 0 && tid < 16) me.codes_out[(size_t)s.bst[ST_EMIT][v.b] * 16 + tid] = (long long)s.codes[tid];
      csync();
      // ---- bookkeeping + max_seq_len rule (generate.py:175-177: the frame is already emitted)
      if (warp == 0) {
        bool r = false;
        if (lane < B && ((run >> lane) & 1u)) {
          s.bst[ST_EMIT][lane] += 1;
          const int pos = P.sl[lane].prefill_len + s.bst[ST_STEP][lane];
          if (pos >= P.max_seq_len - 1) {
            s.bst[ST_FIN][lane] = FQ3_FIN_MAX_SEQ;
            s.bst[ST_STEP][lane] += 1;
          } else {
            r = true;
          }
        }
        const unsigned m = __ballot_sync(0xffffffffu, r);
        if (lane == 0) s.ibc[0] = (int)m;
      }
      csync();
      const uint32_t run2 = (uint32_t)s.ibc[0];
      if (tid == 0) {
        int n = 0;
        for (int b = 0; b < B; ++b)
          if ((run2 >> b) & 1u) s.runl[n++] = b;
        s.runl[32] = n;
      }
      csync();
      if (run2 == 0u) break;
      const bool mine2 = (run2 >> v.b) & 1u;
      // ================= talker step =================
      // layer-0 input: sum of 16 embedding rows + trailing text / tts_pad (generate.py:163-171)
      pmark(c, PC_NORM);
      if (mine2 && v.rank < npt) {
        uint8_t* xn = reinterpret_cast<uint8_t*>(P.XNB) + (size_t)v.b * P.ldX * esz;
        float* xr = P.XB + (size_t)v.b * P.ldX;
        const void* extra = gen_step < me.trailing_len ? me.trailing : me.tts_pad;
        const size_t eoff = gen_step < me.trailing_len ? (size_t)gen_step * Ht : 0;
        norm_row_b<BF>(c, [&](int k) {
          float sm = ldw<BF>(P.t_embed, (size_t)token * Ht + k);
          for (int q = 0; q < P.ncb; ++q) sm += ldw<BF>(P.p_embeds, ((size_t)q * P.p.V + s.codes[q + 1]) * Ht + k);
          return rnd<BF>(rnd<BF>(sm) + ldw<BF>(extra, eoff + k));
        }, P.t.ln_in, 0, Ht, P.t.eps, xn, xr, nullptr, v.rank, npt);
      }
      stack_b<BF, true>(c, P.t, v, 1, run2, 0);
      {
        EpiB e{EP_F32, P.LOGB, nullptr, VMAX, nullptr, 0, nullptr};
        gemv_b<BF>(c, P.t.seg_head, Ht, P.XNB, P.ldX, B, e);
      }
      grid_sync_p(c, PC_SAMPLE);
      if (mine2) {
        const int tok = sample_block<BF>(c, frame_talker_draw(P, me, P.LOGB + (size_t)v.b * VMAX, urow, step,
            // column 0 of the frame just emitted (the bookkeeping above already counted it)
            (me.logprob_out && v.rank == 0) ? me.logprob_out + (size_t)(s.bst[ST_EMIT][v.b] - 1) * 16 : nullptr));
        if (v.rank == 0 && tid == 0) P.TOKB[v.b] = tok;
      }
      grid_sync_p(c, PC_OTHER);
      if (tid < B && ((run2 >> tid) & 1u))
        frame_advance(s.bst[ST_TOKEN][tid], s.bst[ST_STEP][tid], s.bst[ST_GEN][tid], __ldcg(P.TOKB + tid));
      csync();
    }
    pmark(c, PC_OTHER);
    if ((P.dbg_on & 2) && cta == 0 && tid == 0 && P.mode != MODE_GEMV_TEST)
      for (int i = 0; i < PC_N; ++i) reinterpret_cast<long long*>(P.dbg)[i] += s.prof[2 + i];   // accumulates over launches
    if (v.rank == 0 && P.mode != MODE_GEMV_TEST) {
      if (tid == 0)
        put_state(me.state, s.bst[ST_TOKEN][v.b], s.bst[ST_STEP][v.b], s.bst[ST_GEN][v.b], s.bst[ST_FIN][v.b],
                  s.bst[ST_EMIT][v.b]);
      for (int i = tid; i < VMAX / 32; i += NCT) me.seen[i] = s.seen[i];
    }
    drain_producer(c);
  }
  __syncthreads();
}

}  // namespace fq3
