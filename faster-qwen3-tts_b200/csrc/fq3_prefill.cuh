// fq3_prefill.cuh -- K3: hand-written talker prefill (bf16).  Included at the end of fq3_engine.cu.
//
// Replaces the variable-length prompt forward the reference delegates to upstream HF eager code
// (faster_qwen3_tts/generate.py:107-118, streaming.py:63-74) and the 56 index_copy_ calls of
// TalkerGraph.prefill_kv (talker_graph.py:153-170): K and V are written straight into the request's pages of the
// engine's paged talker cache (fq3::kv_row).  Per layer: RMSNorm rows -> QKV GEMM -> q/k-norm + RoPE + KV append ->
// causal GQA attention (eager semantics: bf16 scores, fp32 softmax rounded to bf16, bf16 P.V) -> o_proj GEMM with
// fused residual -> RMSNorm rows -> gate/up GEMM with fused SwiGLU (interleaved columns) -> down GEMM with fused
// residual.  GEMMs are the shared implicit-GEMM tensor-core kernel (fq3gemm::gemm, taps = 1).
//
// Several prompts go through one chain (fq3_prefill_batch; fq3_prefill is its n = 1 case): their rows are packed
// row-major, [sum P_b][H], and the norms and GEMMs run on the packed rows as they are -- a row's result does not depend
// on the rows next to it.  RoPE / KV append and the attention read the sequence table (by value, in the kernel
// parameters) to map a packed row or a query block back to its sequence.  The attention's query blocks and key tiles
// are aligned to each sequence's own row 0 and cache row 0, so every sequence sees exactly the tiles, masks and
// online-softmax order of a launch with that sequence alone: the batch is bit-identical to one prefill per sequence.
#pragma once
#include "fq3_gemm.cuh"

namespace pf {

constexpr int MAXSEQ = 32;   // sequences of one chain (= the engine's request slots)

struct SeqTab {
  int n;                 // sequences
  int row0[MAXSEQ];      // packed row of the sequence's row 0
  int P[MAXSEQ];         // prompt rows
  int pad[MAXSEQ];       // left pad (keys below it are masked, RoPE position = t - pad)
  int slot[MAXSEQ];      // request slot whose KV cache receives rows [0, P)
  int qb0[MAXSEQ + 1];   // first 32-query block of the sequence in the attention grid; qb0[n] = all blocks
};

// the sequence holding packed row r / attention block x (n <= 32: a scan of the parameter table)
__device__ __forceinline__ int seq_of_row(const SeqTab& tab, int r) {
  int b = 0;
  while (b + 1 < tab.n && r >= tab.row0[b + 1]) ++b;
  return b;
}
__device__ __forceinline__ int seq_of_qblock(const SeqTab& tab, int x) {
  int b = 0;
  while (b + 1 < tab.n && x >= tab.qb0[b + 1]) ++b;
  return b;
}

__device__ __forceinline__ float rb(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// one block (256 threads) per row: y = w * rnd(x * rsqrt(mean(x^2) + eps))
__device__ __forceinline__ void rmsnorm_row(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w, int H,
                                            float eps, __nv_bfloat16* __restrict__ y) {
  __shared__ float red[8];
  const int tid = threadIdx.x;
  float v[8];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int k = tid + i * 256;
    v[i] = k < H ? __bfloat162float(x[k]) : 0.f;
    ss += v[i] * v[i];
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if ((tid & 31) == 0) red[tid >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += red[i];
  const float r = 1.0f / sqrtf(tot / (float)H + eps);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int k = tid + i * 256;
    if (k < H) y[k] = __float2bfloat16_rn(__bfloat162float(w[k]) * rb(v[i] * r));
  }
}

// Y[row] = norm(X[row]) for every packed row
__global__ void rmsnorm_rows_kernel(const __nv_bfloat16* __restrict__ X, const __nv_bfloat16* __restrict__ w, int H,
                                    float eps, __nv_bfloat16* __restrict__ Y) {
  fq3gemm::pdl_launch();
  fq3gemm::pdl_wait();
  const size_t row = blockIdx.x;
  rmsnorm_row(X + row * H, w, H, eps, Y + row * H);
}

// Y[b] = norm(last row of sequence b): the final norm, whose rows feed the head GEMM (M = n) and past_hidden
__global__ void rmsnorm_last_rows_kernel(const __nv_bfloat16* __restrict__ X, const __nv_bfloat16* __restrict__ w, int H,
                                         float eps, __nv_bfloat16* __restrict__ Y, const __grid_constant__ SeqTab tab) {
  fq3gemm::pdl_launch();
  fq3gemm::pdl_wait();
  const int b = blockIdx.x;
  rmsnorm_row(X + (size_t)(tab.row0[b] + tab.P[b] - 1) * H, w, H, eps, Y + (size_t)b * H);
}

// one warp per (packed row, vector) with vector in [q heads | k heads | v heads]: q/k RMSNorm + RoPE in place (q) or
// into the KV cache of the row's sequence at its cache row t (k, v).  QKV is [rows][qd + 2 kd] bf16; kv is the page
// pool of the L-layer cache, slot s's page table starts at tabs + s * npt (kv_row).
__global__ void rope_kv_kernel(__nv_bfloat16* __restrict__ QKV, int rows, int nH, int nKV, const __nv_bfloat16* qn,
                               const __nv_bfloat16* kn, const float* __restrict__ cosT, const float* __restrict__ sinT,
                               int npos, float eps, void* kv, const int* __restrict__ tabs, int npt, int L, int layer,
                               const __grid_constant__ SeqTab tab) {
  fq3gemm::pdl_launch();
  fq3gemm::pdl_wait();
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int nvec = nH + 2 * nKV;
  if (gw >= rows * nvec) return;
  const int row = gw / nvec, vi = gw % nvec;
  const int sq = seq_of_row(tab, row);
  const int t = row - tab.row0[sq], n_left_pad = tab.pad[sq];
  const int ld = (nH + 2 * nKV) * 128;
  __nv_bfloat16* src = QKV + (size_t)row * ld + (size_t)vi * 128;
  float v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = __bfloat162float(src[lane + 32 * i]);
  const int what = vi < nH ? 0 : (vi < nH + nKV ? 1 : 2);
  if (what < 2) {
    float ss = v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3];
#pragma unroll
    for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float r = 1.0f / sqrtf(ss / 128.0f + eps);
    const __nv_bfloat16* nw = what == 0 ? qn : kn;
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = rb(__bfloat162float(nw[lane + 32 * i]) * rb(v[i] * r));
    int rp = t - n_left_pad;
    rp = rp < 0 ? 0 : (rp >= npos ? npos - 1 : rp);
    float o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = lane + 32 * i;
      const float cc = rb(cosT[(size_t)rp * 128 + e]), sv = rb(sinT[(size_t)rp * 128 + e]);
      const float rot = (i < 2) ? -v[i + 2] : v[i - 2];
      o[i] = rb(rb(v[i] * cc) + rb(rot * sv));
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = o[i];
  }
  if (what == 0) {
#pragma unroll
    for (int i = 0; i < 4; ++i) src[lane + 32 * i] = __float2bfloat16_rn(v[i]);
  } else {
    const int g = what == 1 ? vi - nH : vi - nH - nKV;
    __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(
        fq3::kv_row(kv, L, nKV, 2, tabs + (size_t)tab.slot[sq] * npt, what - 1, layer, g, t));
#pragma unroll
    for (int i = 0; i < 4; ++i) dst[lane + 32 * i] = __float2bfloat16_rn(v[i]);
  }
}

// ------------------------------------------------------------------------------------------------------------
// Tensor-core causal GQA attention for the prompt (mma.sync m16n8k16, online softmax).  Block = 4 warps = the REP
// q-heads of ONE kv group x two 16-query tiles, so the group's K / V rows are staged once (cp.async, double-buffered
// 32-key tiles, XOR-swizzled for ldmatrix) for all of them.  Rounding points of the eager reference that survive: the
// scores are rounded to bf16, scaled and rounded again; probabilities enter P.V as bf16; the output is bf16.  The
// softmax is the online (running max / running sum) form in fp32, i.e. probabilities are rounded relative to the
// running maximum instead of the final one -- within the bf16 envelope the parity test states.
//   grid = (tab.qb0[tab.n], nKV): blockIdx.x is query block qb of sequence b, qb0[b] + qb, whose rows are counted
//   from the sequence's row 0 and whose key tiles from its cache row 0 -- the tiles of a launch with b alone.  Keys
//   below the sequence's pad are masked; rows below it produce zeros.
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void ldsm_x4(uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "r"((uint32_t)__cvta_generic_to_shared(p)));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "r"((uint32_t)__cvta_generic_to_shared(p)));
}
__device__ __forceinline__ void mma_16816(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&v);
}

template <int REP>
__global__ void __launch_bounds__(128) attn_prefill_mma_kernel(const __nv_bfloat16* __restrict__ QKVp, int nH, int nKV,
                                                              void* kv, const int* __restrict__ tabs, int npt, int L,
                                                              int layer, __nv_bfloat16* __restrict__ OUTp,
                                                              const __grid_constant__ SeqTab tab) {
  constexpr int KT = 32;                                   // keys per staged tile
  __shared__ __align__(128) uint8_t sm[2][2][KT * 256];    // [buffer][K | V][key row x 256 B], 16-byte chunks XOR-swizzled
  fq3gemm::pdl_launch();
  fq3gemm::pdl_wait();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int gq = lane >> 2, t = lane & 3;
  const int sq = seq_of_qblock(tab, blockIdx.x);
  const int g = blockIdx.y, qb = blockIdx.x - tab.qb0[sq];
  const int P = tab.P[sq], n_left_pad = tab.pad[sq];
  const int ld = (nH + 2 * nKV) * 128;
  const __nv_bfloat16* QKV = QKVp + (size_t)tab.row0[sq] * ld;
  __nv_bfloat16* OUT = OUTp + (size_t)tab.row0[sq] * nH * 128;
  const bool active = warp < 2 * REP;
  const int h = g * REP + (warp % REP);
  const int q0 = qb * 32 + (warp / REP) * 16;
  const int i0 = q0 + gq, i1 = q0 + gq + 8;
  const int* pages = tabs + (size_t)tab.slot[sq] * npt;
  const int kt_first = n_left_pad / KT;
  const int kt_last = min(qb, (P - 1) / KT);

  auto load_tile = [&](int kt, int buf) {
    const int k0 = kt * KT;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = tid + 128 * i;
      const int mat = idx >> 9, r = (idx & 511) >> 4, ch = idx & 15;
      const int key = k0 + r;
      const bool ok = key < P;
      // a 32-key tile never straddles a KV_PAGE-row page
      const __nv_bfloat16* src =
          reinterpret_cast<const __nv_bfloat16*>(fq3::kv_row(kv, L, nKV, 2, pages, mat, layer, g, ok ? key : 0)) + ch * 8;
      fq3gemm::cp_async16(&sm[buf][mat][r * 256 + ((ch ^ (r & 7)) << 4)], src, ok);
    }
  };

  // Q fragments of this warp's 16 queries (A operand, 8 k-steps of 16 dims)
  uint32_t qf[8][4];
  if (active) {
    const __nv_bfloat16* qr0 = QKV + (size_t)min(i0, P - 1) * ld + h * 128;
    const __nv_bfloat16* qr1 = QKV + (size_t)min(i1, P - 1) * ld + h * 128;
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      qf[ks][0] = *reinterpret_cast<const uint32_t*>(qr0 + ks * 16 + 2 * t);
      qf[ks][1] = *reinterpret_cast<const uint32_t*>(qr1 + ks * 16 + 2 * t);
      qf[ks][2] = *reinterpret_cast<const uint32_t*>(qr0 + ks * 16 + 8 + 2 * t);
      qf[ks][3] = *reinterpret_cast<const uint32_t*>(qr1 + ks * 16 + 8 + 2 * t);
    }
  }
  float oacc[16][4];
#pragma unroll
  for (int n = 0; n < 16; ++n)
#pragma unroll
    for (int r = 0; r < 4; ++r) oacc[n][r] = 0.f;
  float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f};
  const float scale = 0.08838834764831845f;  // 128^-0.5

  if (kt_first <= kt_last) {
    load_tile(kt_first, 0);
    fq3gemm::cp_commit();
  }
  int buf = 0;
  for (int kt = kt_first; kt <= kt_last; ++kt, buf ^= 1) {
    if (kt + 1 <= kt_last) {
      load_tile(kt + 1, buf ^ 1);
      fq3gemm::cp_commit();
      fq3gemm::cp_wait<1>();
    } else {
      fq3gemm::cp_wait<0>();
    }
    __syncthreads();
    if (active) {
      const uint8_t* Ks = sm[buf][0];
      const uint8_t* Vs = sm[buf][1];
      const int k0 = kt * KT;
      // ---- S = Q K^T for the 32 keys of the tile
      float sacc[4][4];
#pragma unroll
      for (int n = 0; n < 4; ++n)
#pragma unroll
        for (int r = 0; r < 4; ++r) sacc[n][r] = 0.f;
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
#pragma unroll
        for (int np = 0; np < 2; ++np) {   // n-tiles 2np, 2np + 1
          const int m = lane >> 3, r = lane & 7;
          const int row = (2 * np + (m >> 1)) * 8 + r, ch = 2 * ks + (m & 1);
          uint32_t b0, b1, b2, b3;
          ldsm_x4(b0, b1, b2, b3, Ks + row * 256 + ((ch ^ (row & 7)) << 4));
          mma_16816(sacc[2 * np], qf[ks], b0, b1);
          mma_16816(sacc[2 * np + 1], qf[ks], b2, b3);
        }
      }
      // ---- mask, bf16 rounding points, online softmax (rows i0: c0,c1 ; i1: c2,c3)
      float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int n = 0; n < 4; ++n)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int j = k0 + n * 8 + 2 * t + (r & 1);
          const int i = (r < 2) ? i0 : i1;
          const bool ok = j <= i && j >= n_left_pad && j < P;
          const float sv = ok ? rb(rb(sacc[n][r]) * scale) : -INFINITY;
          sacc[n][r] = sv;
          tmax[r >> 1] = fmaxf(tmax[r >> 1], sv);
        }
      float corr[2], mnew[2];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        tmax[rr] = fmaxf(tmax[rr], __shfl_xor_sync(0xffffffffu, tmax[rr], 1));
        tmax[rr] = fmaxf(tmax[rr], __shfl_xor_sync(0xffffffffu, tmax[rr], 2));
        mnew[rr] = fmaxf(mrow[rr], tmax[rr]);
        corr[rr] = (mrow[rr] == -INFINITY) ? 0.f : expf(mrow[rr] - mnew[rr]);
        mrow[rr] = mnew[rr];
      }
      float psum[2] = {0.f, 0.f};
      uint32_t pf[4][2];   // bf16 pairs: [n-tile][row half]
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        float pv[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const float mm = mnew[r >> 1];
          pv[r] = (sacc[n][r] == -INFINITY || mm == -INFINITY) ? 0.f : rb(expf(sacc[n][r] - mm));
          psum[r >> 1] += pv[r];
        }
        pf[n][0] = pack_bf16(pv[0], pv[1]);
        pf[n][1] = pack_bf16(pv[2], pv[3]);
      }
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        psum[rr] += __shfl_xor_sync(0xffffffffu, psum[rr], 1);
        psum[rr] += __shfl_xor_sync(0xffffffffu, psum[rr], 2);
        lrow[rr] = lrow[rr] * corr[rr] + psum[rr];
      }
#pragma unroll
      for (int n = 0; n < 16; ++n) {
        oacc[n][0] *= corr[0]; oacc[n][1] *= corr[0];
        oacc[n][2] *= corr[1]; oacc[n][3] *= corr[1];
      }
      // ---- O += P V  (two k-steps of 16 keys, 16 n-tiles of 8 dims)
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        const uint32_t a[4] = {pf[2 * kk][0], pf[2 * kk][1], pf[2 * kk + 1][0], pf[2 * kk + 1][1]};
#pragma unroll
        for (int dn = 0; dn < 8; ++dn) {
          const int m = lane >> 3, r = lane & 7;
          const int row = 16 * kk + (m & 1) * 8 + r, ch = 2 * dn + (m >> 1);
          uint32_t b0, b1, b2, b3;
          ldsm_x4_t(b0, b1, b2, b3, Vs + row * 256 + ((ch ^ (row & 7)) << 4));
          mma_16816(oacc[2 * dn], a, b0, b1);
          mma_16816(oacc[2 * dn + 1], a, b2, b3);
        }
      }
    }
    __syncthreads();   // everyone is done with `buf` before the next iteration's prefetch overwrites it
  }
  if (!active) return;
  const float inv0 = lrow[0] > 0.f ? 1.0f / lrow[0] : 0.f, inv1 = lrow[1] > 0.f ? 1.0f / lrow[1] : 0.f;
#pragma unroll
  for (int n = 0; n < 16; ++n) {
    if (i0 < P)
      *reinterpret_cast<uint32_t*>(OUT + (size_t)i0 * nH * 128 + h * 128 + n * 8 + 2 * t) = pack_bf16(oacc[n][0] * inv0, oacc[n][1] * inv0);
    if (i1 < P)
      *reinterpret_cast<uint32_t*>(OUT + (size_t)i1 * nH * 128 + h * 128 + n * 8 + 2 * t) = pack_bf16(oacc[n][2] * inv1, oacc[n][3] * inv1);
  }
}

}  // namespace pf

static int pf_gemm(fq3_engine* e, const __nv_bfloat16* X, const __nv_bfloat16* W, const __nv_bfloat16* R,
                   __nv_bfloat16* Y, int T, int K, int N, int mode, cudaStream_t stream) {
  fq3gemm::ConvArgs a;
  memset(&a, 0, sizeof(a));
  a.X = X; a.W = W; a.R = R; a.Yraw = Y; a.T = T; a.Cin = K; a.N = N; a.taps = 1; a.dil = 1;
  a.bias_mod = 1; a.act_mod = 1; a.mode = mode;
  e->launches++;
  if (const char* err = fq3gemm::gemm(a, stream)) return fail(FQ3_ERR_CUDA, "prefill GEMM: %s", err);
  return 0;
}

extern "C" int fq3_engine_set_prefill_weights(fq3_engine* e, const fq3_tensor* tensors, int32_t n) {
  if (!e || !tensors) return fail(FQ3_ERR_INVALID, "null argument");
  if (!e->bf16) return fail(FQ3_ERR_INVALID, "the hand-written prefill is bf16 only");
  const fq3_stack_config& T = e->cfg.talker;
  const int64_t L = T.num_hidden_layers, H = T.hidden_size, I = T.intermediate_size;
  const int64_t qd = T.num_attention_heads * 128, kd = T.num_key_value_heads * 128;
  struct Want { const char* nm; int64_t numel; const void** dst; } want[] = {
      {"t.qkv", L * (qd + 2 * kd) * H, &e->pf_qkv}, {"t.o", L * H * qd, &e->pf_o}, {"t.gu", L * 2 * I * H, &e->pf_gu},
      {"t.down", L * H * I, &e->pf_down}, {"t.head", (int64_t)T.vocab_size * H, &e->pf_head}};
  for (auto& w : want) {
    *w.dst = nullptr;
    for (int i = 0; i < n; ++i)
      if (!strcmp(tensors[i].name, w.nm)) {
        if (tensors[i].numel != w.numel) return fail(FQ3_ERR_INVALID, "prefill tensor '%s': bad numel", w.nm);
        if ((uintptr_t)tensors[i].dev_ptr & 15) return fail(FQ3_ERR_INVALID, "prefill tensor '%s' is not 16-byte aligned", w.nm);
        *w.dst = tensors[i].dev_ptr;
      }
    if (!*w.dst) return fail(FQ3_ERR_INVALID, "missing prefill tensor '%s'", w.nm);
  }
  if (H > 2048 || H % 32 || I % 32) return fail(FQ3_ERR_INVALID, "prefill geometry unsupported");
  const int nH = T.num_attention_heads, nKV = T.num_key_value_heads;
  if (nH != nKV && nH != 2 * nKV)
    return fail(FQ3_ERR_INVALID, "prefill: talker GQA ratio num_attention_heads / num_key_value_heads = %d / %d is "
                "unsupported (the prefill attention takes ratios 1 and 2)", nH, nKV);
  if (T.vocab_size % 8)
    return fail(FQ3_ERR_INVALID, "prefill: talker vocab_size %d is not a multiple of 8 (N of the head GEMM)", T.vocab_size);
  DevGuard dev_guard(e->dev);
  const size_t S = e->cfg.max_seq_len;
  const size_t wide = std::max<size_t>(qd + 2 * kd, (size_t)I);
  if (!e->pf_buf[0]) {
    CK(cudaMalloc(&e->pf_buf[0], S * H * 2));      // x
    CK(cudaMalloc(&e->pf_buf[1], S * H * 2));      // x1
    CK(cudaMalloc(&e->pf_buf[2], S * H * 2));      // normed
    CK(cudaMalloc(&e->pf_buf[3], S * wide * 2));   // qkv / act
    CK(cudaMalloc(&e->pf_buf[4], S * qd * 2));     // attention out
  }
  e->pf_ready = true;
  return 0;
}

// One chain of launches over the sequences of `tab` (sum of P <= max_seq_len rows): embeds [rows][H] packed as the table
// says -> KV caches of the listed slots, logits [n][V], hidden [n][H].
static int prefill_group(fq3_engine* e, const pf::SeqTab& tab, const void* embeds_dev, void* logits_out_dev,
                         void* hidden_out_dev, cudaStream_t stream) {
  const fq3_stack_config& T = e->cfg.talker;
  const int L = T.num_hidden_layers, H = T.hidden_size, I = T.intermediate_size;
  const int nH = T.num_attention_heads, nKV = T.num_key_value_heads, qd = nH * 128, kd = nKV * 128;
  const int rows = tab.row0[tab.n - 1] + tab.P[tab.n - 1], n = tab.n;
  using bf = __nv_bfloat16;
  bf* x = (bf*)e->pf_buf[0];
  bf* x1 = (bf*)e->pf_buf[1];
  bf* hn = (bf*)e->pf_buf[2];
  bf* wide = (bf*)e->pf_buf[3];
  bf* att = (bf*)e->pf_buf[4];
  CK(cudaMemcpyAsync(x, embeds_dev, (size_t)rows * H * 2, cudaMemcpyDeviceToDevice, stream));
  const KParams& k = e->kp;
  int rc;
  for (int l = 0; l < L; ++l) {
    FQ3_LAUNCH((pf::rmsnorm_rows_kernel), rows, 256, 0, stream, x, (const bf*)k.t.ln_in + (size_t)l * H, H, T.rms_norm_eps, hn);
    e->launches++;
    if ((rc = pf_gemm(e, hn, (const bf*)e->pf_qkv + (size_t)l * (qd + 2 * kd) * H, nullptr, wide, rows, H, qd + 2 * kd, 0, stream))) return rc;
    {
      const int warps = rows * (nH + 2 * nKV);
      FQ3_LAUNCH((pf::rope_kv_kernel), (warps * 32 + 255) / 256, 256, 0, stream,
          wide, rows, nH, nKV, (const bf*)k.t.qnorm + (size_t)l * 128, (const bf*)k.t.knorm + (size_t)l * 128, k.t.cos,
          k.t.sin, k.t.npos, T.rms_norm_eps, e->kv, e->kv_tab, e->kv_npt, L, l, tab);
      e->launches++;
    }
    if (nH == 2 * nKV)   // fq3_engine_set_prefill_weights admits GQA ratios 1 and 2 only
      FQ3_LAUNCH((pf::attn_prefill_mma_kernel<2>), dim3(tab.qb0[n], nKV), 128, 0, stream, wide, nH, nKV, e->kv, e->kv_tab, e->kv_npt, L, l, att, tab);
    else
      FQ3_LAUNCH((pf::attn_prefill_mma_kernel<1>), dim3(tab.qb0[n], nKV), 128, 0, stream, wide, nH, nKV, e->kv, e->kv_tab, e->kv_npt, L, l, att, tab);
    e->launches++;
    if ((rc = pf_gemm(e, att, (const bf*)e->pf_o + (size_t)l * H * qd, x, x1, rows, qd, H, 0, stream))) return rc;
    FQ3_LAUNCH((pf::rmsnorm_rows_kernel), rows, 256, 0, stream, x1, (const bf*)k.t.ln_post + (size_t)l * H, H, T.rms_norm_eps, hn);
    e->launches++;
    if ((rc = pf_gemm(e, hn, (const bf*)e->pf_gu + (size_t)l * 2 * I * H, nullptr, wide, rows, H, 2 * I, 1, stream))) return rc;
    if ((rc = pf_gemm(e, wide, (const bf*)e->pf_down + (size_t)l * H * I, x1, x, rows, I, H, 0, stream))) return rc;
  }
  // final norm of every sequence's last row -> past_hidden; logits = codec_head(hidden), M = n
  FQ3_LAUNCH((pf::rmsnorm_last_rows_kernel), n, 256, 0, stream, x, (const bf*)k.t.ln_f, H, T.rms_norm_eps, hn, tab);
  e->launches++;
  CK(cudaMemcpyAsync(hidden_out_dev, hn, (size_t)n * H * 2, cudaMemcpyDeviceToDevice, stream));
  if ((rc = pf_gemm(e, hn, (const bf*)e->pf_head, nullptr, (bf*)logits_out_dev, n, H, T.vocab_size, 0, stream))) return rc;
  CK(cudaGetLastError());
  return 0;
}

extern "C" int fq3_prefill_batch(fq3_engine* e, int32_t n, const int32_t* slots, const void* embeds_dev, const int32_t* P,
                                 const int32_t* n_left_pad, void* logits_out_dev, void* hidden_out_dev, void* stream_) {
  if (!e) return fail(FQ3_ERR_INVALID, "null argument");
  if (n < 1 || n > e->max_batch) return fail(FQ3_ERR_INVALID, "n %d outside [1, max_batch=%d] (prompts of one call)", n, e->max_batch);
  if (!slots || !embeds_dev || !P || !n_left_pad || !logits_out_dev || !hidden_out_dev) return fail(FQ3_ERR_INVALID, "null argument");
  // every check before the first launch: a refused call leaves every slot as it was.  A row is named when n > 1.
  char row[32] = "";
  for (int i = 0; i < n; ++i) {
    if (n > 1) snprintf(row, sizeof(row), " (row %d)", i);
    if (slots[i] < 0 || slots[i] >= e->max_slots)
      return fail(FQ3_ERR_INVALID, "slot %d outside [0, %s=%d)%s", slots[i], slot_bound(e), e->max_slots, row);
    for (int j = 0; j < i; ++j)
      if (slots[j] == slots[i]) return fail(FQ3_ERR_INVALID, "slot %d listed twice%s", slots[i], row);
    if (P[i] <= 0) return fail(FQ3_ERR_INVALID, "empty prompt%s", row);
    if (P[i] > e->cfg.max_seq_len)
      return fail(FQ3_ERR_TOO_LONG, "Input is too long: prefill has %d tokens but max_seq_len=%d. Use shorter text or shorter reference audio.%s", P[i], e->cfg.max_seq_len, row);
    int rc;
    if ((rc = check_rows(e, slots[i], P[i], "the prompt"))) return rc;
  }
  if (!e->pf_ready) return fail(FQ3_ERR_STATE, "fq3_engine_set_prefill_weights has not been called");
  if ((uintptr_t)logits_out_dev & 15) return fail(FQ3_ERR_INVALID, "logits_out_dev must be 16-byte aligned");
  DevGuard dev_guard(e->dev);
  cudaStream_t stream = (cudaStream_t)stream_;
  const int H = e->cfg.talker.hidden_size, V = e->cfg.talker.vocab_size;
  // consecutive groups in the caller's order, each as many sequences as fit the max_seq_len rows of scratch
  size_t in_row = 0;
  for (int b0 = 0; b0 < n;) {
    pf::SeqTab tab;
    memset(&tab, 0, sizeof(tab));
    int rows = 0, qb = 0;
    while (b0 + tab.n < n && rows + P[b0 + tab.n] <= e->cfg.max_seq_len) {
      const int i = b0 + tab.n, j = tab.n++;
      tab.row0[j] = rows; tab.P[j] = P[i]; tab.pad[j] = n_left_pad[i]; tab.slot[j] = slots[i]; tab.qb0[j] = qb;
      rows += P[i];
      qb += (P[i] + 31) / 32;
    }
    tab.qb0[tab.n] = qb;
    int rc;
    if ((rc = prefill_group(e, tab, (const __nv_bfloat16*)embeds_dev + in_row * H,
                            (__nv_bfloat16*)logits_out_dev + (size_t)b0 * V, (__nv_bfloat16*)hidden_out_dev + (size_t)b0 * H,
                            stream)))
      return rc;
    in_row += rows;
    b0 += tab.n;
  }
  return 0;
}

extern "C" int fq3_prefill(fq3_engine* e, int32_t slot, const void* embeds_dev, int32_t P, int32_t n_left_pad,
                           void* logits_out_dev, void* hidden_out_dev, void* stream) {
  return fq3_prefill_batch(e, 1, &slot, embeds_dev, &P, &n_left_pad, logits_out_dev, hidden_out_dev, stream);
}
