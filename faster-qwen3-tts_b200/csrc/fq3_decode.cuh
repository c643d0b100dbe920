// fq3_decode.cuh -- the persistent decode kernel (sm_90a).
//
// One cooperative launch runs a whole chunk of codec frames on device: per frame the 15-pass code predictor
// (reference: faster_qwen3_tts/predictor_graph.py:115-167), the 16-row embedding sum (generate.py:163-171), the
// 28-layer talker step (talker_graph.py:97-107,198-214), codec_head, repetition penalty and sampling
// (generate.py:182-197, sampling.py:10-66) and the EOS / max-length control flow (generate.py:149-151,175-177).
// No per-token launch, graph replay or host round trip remains inside a chunk.
//
// Structure of a CTA (one per SM, 288 threads):
//   warp 8      PRODUCER: walks this CTA's slice of the weight "tape" (weights pre-packed at load time into
//               the exact order they are consumed) and streams it with cp.async.bulk (TMA bulk copy, SASS
//               UBLKCP) into a 5 x 32 KB shared-memory ring guarded by full/empty mbarriers.  It never takes
//               part in grid barriers, so HBM keeps streaming while the consumers synchronise / do attention.
//   warps 0..7  CONSUMERS: fp32-accumulate GEMV rows straight out of the ring (conflict-free 16-byte LDS),
//               warp-shuffle reductions, fused epilogues (residual add, SiLU*up, bias), RMSNorm prologues,
//               GQA attention over the KV cache, and block-wide sampling.  Everything that is cheap is
//               computed redundantly in every CTA (norms, sampling, embedding sums) so that only five grid
//               barriers per layer remain.
//
// Numerics follow the reference's eager bf16 / fp32 rounding points (template parameter BF): products of
// dtype-rounded operands are accumulated in fp32 and rounded to the model dtype wherever torch would
// materialise a tensor.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/fq3_engine.h"   // enum fq3_finish: the finish codes the kernels write
#include "fq3_tape.cuh"                  // the weight tape: Grp, segment table, STAGE_BYTES

namespace fq3 {

constexpr int NCW = 8;               // consumer warps
constexpr int NCT = NCW * 32;        // consumer threads
constexpr int NTHREADS = NCT + 32;   // + producer warp
constexpr int NS = 5;                // ring stages
constexpr int XS_FLOATS = 6144;      // activation vector(s) feeding the current GEMV; also attention/sampling scratch
constexpr int HMAX = 2048;           // max talker hidden (xin / past_hidden buffers)
constexpr int VMAX = 4096;
constexpr int SEQMAX = 4096;

enum Mode { MODE_FUSED = 0, MODE_TALKER_STEP = 1, MODE_PRED_RUN = 2, MODE_GEMV_TEST = 3 };

// split-key talker attention runs from this many cached keys on (below, one CTA per q-head is faster); run_layers and
// Producer::stack_layers must take the same decision, so both read this one constant
constexpr int ATTN_SPLIT_MIN = 192;

struct Sampling {
  int do_sample, top_k;
  float temperature, top_p, penalty;
};

struct StackDev {
  int H, I, L, nH, nKV, V, qd, kd, rep;
  float eps;
  int seg_base;        // segment id of layer 0 / QKV; layer l uses seg_base + 4*l + {0:QKV,1:O,2:GU,3:DN}
  int seg_head;        // first head segment
  const void *ln_in, *ln_post, *qnorm, *knorm, *ln_f;
  int S;               // predictor: cache rows per kv head, [L][nKV][S][128] model dtype (the talker's cache is paged)
  const float *cos, *sin;  // [npos][128] fp32
  int npos;
};

// ---- talker KV cache: pages of KV_PAGE rows from one engine-wide pool.  Page p is ONE contiguous block
// {K [L][nKV][KV_PAGE][128], V [L][nKV][KV_PAGE][128]} in model dtype, so the KV_PAGE rows of one (layer, kv head) are
// contiguous.  A slot's page table maps its row block t / KV_PAGE to a page (-1 = unmapped; the engine refuses work
// that would touch such a row before launching it).  kv_row() is the only code that turns a cache row into an address:
// every reader and writer, device (decode, prefill) and host (import / export), goes through it.
constexpr int KV_PAGE = 64;
__host__ __device__ __forceinline__ size_t kv_half_bytes(int L, int nKV, size_t esz) {   // K (or V) part of a page
  return (size_t)L * nKV * KV_PAGE * 128 * esz;
}
// which: 0 = K, 1 = V; row t of (layer, kv head g) of the slot whose table is `pages`
__host__ __device__ __forceinline__ uint8_t* kv_row(void* pool, int L, int nKV, size_t esz, const int* pages, int which,
                                                    int layer, int g, int t) {
  const int page = pages[t / KV_PAGE];   // the kernels pass their copy in shared memory (Smem::kvtab)
  const size_t half = kv_half_bytes(L, nKV, esz);
  return reinterpret_cast<uint8_t*>(pool) + (size_t)page * 2 * half + (size_t)which * half +
         ((size_t)(layer * nKV + g) * KV_PAGE + t % KV_PAGE) * 128 * esz;
}

// a request's loop state: the words of SlotParams::state (and of Smem::bst, the batched kernel's copy).  finished holds
// an fq3_finish code; emitted counts the frames of the last launch.
enum StateWord { ST_TOKEN = 0, ST_STEP = 1, ST_GEN = 2, ST_FIN = 3, ST_EMIT = 4, ST_WORDS = 5 };

// one request: its caches, decode state and parameters.  The single-sequence kernel reads it from KParams::req, the
// batched kernel one per column from KParams::sl.
struct SlotParams {
  void* kv;             // the engine's talker KV page pool (kv_row)
  const int* kv_pages;  // this slot's page table [ceil(max_seq_len / KV_PAGE)]
  void *pkc, *pvc;      // predictor KV cache of this slot [Lp][nKVp][32][128]
  int* state;           // [ST_WORDS] StateWord
  float* past_hidden;   // [HMAX] fp32 holding dtype-rounded values
  uint32_t* seen;       // [VMAX/32] bitmap of cb0 history (sampling.py:22 unique())
  const void* trailing;
  const void* tts_pad;
  const float* uniforms;
  long long* codes_out; // [n_frames][16]
  float* logprob_out;   // [n_frames][16] or nullptr: col k >= 1 = codebook k of the frame, col 0 = the cb0 sampled after it
  int prefill_len, rope_delta, n_left_pad, max_new, min_new, trailing_len;
  int text_open;        // more trailing rows may follow: a frame that would read row >= trailing_len waits (stops the slot)
  int n_frames;         // frames this request may emit in the launch
  Sampling sp_t, sp_p;
};

struct KParams {
  StackDev t, p;
  int mode, ncta, nseg, seg_mtp;
  const uint8_t* tape;
  const Grp* grps;
  const uint32_t* segtab;       // [cta][nseg] seg_begin / seg_count words
  const uint32_t* cta_grp_off;  // [ncta + 1]
  float *X, *X1, *QKV, *LOGITS;
  void* ATT;                    // model dtype: the talker attention output that feeds o_proj
  void* ACT;                    // model dtype [2][ldACT]: SiLU(gate) * up, the down projection's input
  int ldX, ldQKV, ldATT, ldACT;
  unsigned* bar;
  int* xerr;                    // sticky: set when a tagged exchange wait gave up (never cleared by a launch)
  const void* t_embed;
  const void* p_embeds;
  const void* mtp_b;
  const void* mtp_tab;   // [ncb][Vp][Hp] = mtp(embeds[i][code]) precomputed at load time (has_mtp only)
  int has_mtp, ncb, eos, max_seq_len;
  SlotParams req;        // single-sequence kernel: the request of this launch
  int n_frames;          // MODE_FUSED: the producer's frame bound (no request of the launch runs longer)
  const void* in_embeds;
  void* hidden_out;
  int position;
  const void* pred_input;
  const float* pred_uniforms;
  float* dbg;
  int dbg_on;
  long long dbg_stride_layer;  // floats per layer record
  int attn_split;              // talker attention: CTAs per q-head (keys split across them, K/V slices TMA-staged); 0 = off
  float* PART;                 // [nH][attn_split][PART_STRIDE] partial attention results (acc[128], max, sum)
  unsigned* attn_cnt;          // [nH] arrival counters of the splits (cleared with the barrier words every launch)
  // ---- batched decode (fq3_decode_batch.cuh): B request slots share one pass over the weight tape
  int nslots;                  // columns of this launch (0: single-sequence kernel)
  const SlotParams* sl;        // [nslots] per-column request state (device)
  float *XB, *X1B, *QKVB, *LOGB;   // fp32 [MAXCOL][ldX] / [MAXCOL][ldX] / [MAXCOL][ldQKV] / [MAXB][VMAX]
  void *XNB, *ATTB, *ACTB, *PINB;  // model dtype GEMV inputs [MAXCOL][ldX] / [ldATT] / [ldACT] / [HMAX]
  int* TOKB;                   // [MAXB] cb0 token of every column after the talker sampling step
  // MODE_GEMV_TEST: one batched GEMV over segment `gt_seg` (numerics test of the GEMV against a torch reference)
  int gt_seg, gt_K, gt_ncols, gt_rows, gt_swiglu;
  const void* gt_x;            // model dtype [gt_ncols][gt_K]
  void* gt_out;                // fp32 [gt_ncols][gt_rows]  (gt_swiglu: model dtype [gt_ncols][gt_rows / 2])
};

// ------------------------------------------------------------------------------------------------------------
// PTX helpers
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t cnt) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(cnt) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* b) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* b, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(b)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t parity) {
  while (!mbar_try_wait(b, parity)) {
  }
}
// TMA bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_g2s_hint(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t pol) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
      : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void csync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }  // consumers only

// ---- tagged activation exchange (bf16 single-sequence kernel, DESIGN §4).  Every word of QKV, X1, X and LOGITS is an
// fp32 word holding a bf16-rounded value, so its low 16 bits are zero; a producer stores bits(v) | tag and a consumer
// polls the words it needs until their low half equals the exchange's tag, then masks it off.  No counter, no release
// fence and no second load of the vector.  Tags count exchanges from 1 in every launch (the engine clears the four
// buffers with the barrier words before each launch) and skip 0 when they wrap.
constexpr uint32_t XTAG = 0xffffu;
constexpr uint32_t XWAIT_CAP = 1u << 24;   // polls of one word before the launch gives up on it (seconds, not microseconds)
__device__ __forceinline__ uint32_t xtag_next(uint32_t t) { return t == XTAG ? 1u : t + 1u; }
__device__ __forceinline__ float untag(uint32_t w) { return __uint_as_float(w & ~XTAG); }
__device__ __forceinline__ void st_tagged(float* p, float v, uint32_t tag) {   // v: bf16-rounded
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(__float_as_uint(v) | tag) : "memory");
}
__device__ __forceinline__ uint32_t ld_relaxed_u32(const void* p) {
  uint32_t v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint4 ld_relaxed_v4(const void* p) {
  uint4 v;
  asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
// a wait that passes XWAIT_CAP polls is a protocol bug: it sets *err (the engine turns it into an error return) and
// gives up, so the launch runs to its end instead of hanging the GPU; once *err is set, every other wait gives up too
__device__ __noinline__ bool xwait_give_up(int* err, uint32_t n) {
  if (n >= XWAIT_CAP) {
    atomicOr(err, 1);
    return true;
  }
  return ld_relaxed_u32(err) != 0;
}
__device__ __forceinline__ bool xtag_ok(uint32_t w, uint32_t tag) { return (w & XTAG) == tag; }
__device__ __forceinline__ bool xtag_ok(const uint4& w, uint32_t tag) {
  return xtag_ok(w.x, tag) & xtag_ok(w.y, tag) & xtag_ok(w.z, tag) & xtag_ok(w.w, tag);
}
// w: a word (or 16-byte vector) already loaded from p; re-polls p alone, with a growing back-off, until it carries tag
template <class W>
__device__ __forceinline__ W xwait(int* err, const void* p, W w, uint32_t tag) {
  uint32_t ns = 32, n = 0;
  while (!xtag_ok(w, tag)) {
    if ((++n & 1023u) == 0u && xwait_give_up(err, n)) break;
    __nanosleep(ns);
    ns = ns < 256 ? 2 * ns : ns;
    if constexpr (sizeof(W) == 16) w = ld_relaxed_v4(p);
    else w = ld_relaxed_u32(p);
  }
  return w;
}
// one polled word / 16-byte vector of an exchanged buffer, tag masked off
__device__ __forceinline__ float xload(int* err, const float* p, uint32_t tag) {
  uint32_t w = ld_relaxed_u32(p);
  if (!xtag_ok(w, tag)) w = xwait(err, p, w, tag);
  return untag(w);
}
__device__ __forceinline__ float4 xload4(int* err, const float* p, uint32_t tag) {
  uint4 w = ld_relaxed_v4(p);
  if (!xtag_ok(w, tag)) w = xwait(err, p, w, tag);
  return make_float4(untag(w.x), untag(w.y), untag(w.z), untag(w.w));
}

template <bool BF>
__device__ __forceinline__ float rnd(float x) {
  if constexpr (BF)
    return __bfloat162float(__float2bfloat16_rn(x));
  else
    return x;
}
template <bool BF>
__device__ __forceinline__ float ldw(const void* p, size_t i) {  // read-only weight / table element
  if constexpr (BF)
    return __bfloat162float(__ldg(reinterpret_cast<const __nv_bfloat16*>(p) + i));
  else
    return __ldg(reinterpret_cast<const float*>(p) + i);
}
template <bool BF>
__device__ __forceinline__ void stw(void* p, size_t i, float v) {
  if constexpr (BF)
    reinterpret_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(v);
  else
    reinterpret_cast<float*>(p)[i] = v;
}
// an exchanged fp32 activation word: bf16 stores it tagged, fp32 (all 32 bits in use) plainly behind a grid barrier;
// xget reads one that this CTA has already polled, so it only masks the tag
template <bool BF>
__device__ __forceinline__ void xput(float* p, float v, uint32_t tag) {
  if constexpr (BF) st_tagged(p, v, tag);
  else *p = v;
}
template <bool BF>
__device__ __forceinline__ float xget(const float* p) {
  if constexpr (BF) return untag(__float_as_uint(__ldcg(p)));
  else return __ldcg(p);
}
__device__ __forceinline__ float bf_lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf_hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }

// ------------------------------------------------------------------------------------------------------------
// shared memory layout
// ------------------------------------------------------------------------------------------------------------
struct __align__(128) Smem {
  uint8_t ring[NS][STAGE_BYTES];
  float xs[XS_FLOATS];
  float xin[2][HMAX];
  float hid[HMAX];
  Grp grp[MAXGRP];
  uint32_t seg[MAXSEG];
  uint64_t full[NS];
  uint64_t empty[NS];
  float red[NCW];
  int hist[256];
  uint32_t seen[VMAX / 32];
  int codes[16];
  int ibc[4];               // integer broadcast slots
  float fbc[4];             // float broadcast slots
  // hand-shake words between the consumer warps and the producer warp: accessed ONLY through flag_ld / flag_st
  // (shared-memory atomics: well-defined without a block barrier, and silent under compute-sanitizer racecheck)
  int stop_flag;            // consumers -> producer
  int prod_done;            // producer -> consumers
  int prod_issued;          // tiles issued by the producer
  int bst[ST_WORDS][32];    // batched kernel: replicated per-column loop state
  long long prof[12];       // batched kernel, CTA 0 / thread 0: [0] last clock [1] current category [2..] cycles per category
  int runl[36];             // batched kernel: columns running in the current (sub)frame, ascending; [32] = their number
  int kvtab[SEQMAX / KV_PAGE];   // page table of the request being attended to: the single-sequence kernel's, read
                                 // once per launch; the batched kernel's current column, read once per attention item
};

// All dynamic shared memory of the kernel is one Smem; going through this accessor (instead of a reference carried
// in Ctx) lets the compiler prove the address space everywhere: STS/LDS with 32-bit addresses, not generic ST/LD.
extern __shared__ __align__(128) uint8_t fq3_smem_raw[];
__device__ __forceinline__ Smem& SMEM() { return *reinterpret_cast<Smem*>(fq3_smem_raw); }
static_assert(sizeof(Smem) <= 232448, "Smem exceeds the 227 KB per-CTA limit");

__device__ __forceinline__ int flag_ld(int* p) { return atomicAdd(p, 0); }
__device__ __forceinline__ void flag_st(int* p, int v) { atomicExch(p, v); }

struct Ctx {
  const KParams& P;
  int tid, warp, lane;
  uint32_t tile_ctr;   // tiles consumed (identical in every consumer thread)
  unsigned bar_target; // thread 0 only
  uint32_t xtag;       // tag of the latest tagged exchange (identical in every consumer thread of every CTA)
};

// ------------------------------------------------------------------------------------------------------------
// grid barrier (consumer warps of all CTAs).  The producer warp never waits here.
// ------------------------------------------------------------------------------------------------------------
// bar.sync orders the CTA's writes before thread 0's release-reduction (cumulativity); pollers acquire.
__device__ __forceinline__ void grid_sync(Ctx& c) {
  csync();
  if (c.tid == 0) {
    c.bar_target += (unsigned)c.P.ncta;
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(c.P.bar), "r"(1u) : "memory");
    while (ld_acquire_u32(c.P.bar) < c.bar_target) {
    }
  }
  csync();
}

// split form: everything issued between grid_arrive() and grid_wait() overlaps the barrier latency -- used for loads
// that do not depend on other CTAs' results of the current phase (cached K/V rows, norm weights)
__device__ __forceinline__ void grid_arrive(Ctx& c) {
  csync();
  if (c.tid == 0) {
    c.bar_target += (unsigned)c.P.ncta;
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(c.P.bar), "r"(1u) : "memory");
  }
}
__device__ __forceinline__ void grid_wait(Ctx& c) {
  if (c.tid == 0) {
    while (ld_acquire_u32(c.P.bar) < c.bar_target) {
    }
  }
  csync();
}

__device__ __forceinline__ float block_sum(Ctx& c, float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (c.lane == 0) SMEM().red[c.warp] = v;
  csync();
  float r = 0.f;
#pragma unroll
  for (int w = 0; w < NCW; ++w) r += SMEM().red[w];
  csync();
  return r;
}
__device__ __forceinline__ float block_max(Ctx& c, float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  if (c.lane == 0) SMEM().red[c.warp] = v;
  csync();
  float r = SMEM().red[0];
#pragma unroll
  for (int w = 1; w < NCW; ++w) r = fmaxf(r, SMEM().red[w]);
  csync();
  return r;
}

// timing probe (dbg_on & 2): CTA 0 / thread 0 appends clock64() to the tail of the debug buffer
__device__ __forceinline__ void probe(Ctx& c, int& idx) {
  if ((c.P.dbg_on & 2) && blockIdx.x == 0 && c.tid == 0) {
    long long* ts = reinterpret_cast<long long*>(c.P.dbg);
    if (idx < 4096) ts[idx] = clock64();
  }
  idx++;
}

__device__ __forceinline__ void probe_at(Ctx& c, int idx) {  // fixed slot (frame-level phases: slots 1024..)
  if ((c.P.dbg_on & 2) && blockIdx.x == 0 && c.tid == 0)
    reinterpret_cast<long long*>(c.P.dbg)[idx] = clock64();
}

// ------------------------------------------------------------------------------------------------------------
// fp32 GEMV over one segment: rows of this CTA, streamed from the ring.  x: NT vectors of stride xstride, in shared
// memory or (XG) in global memory, read through __ldcg; vectors t >= ncols read vector 0.  (bf16 runs gemv_mma.)
// Epilogue epi(row0, v0[NT], v1[NT]) is called by lane 0 for each row pair (rows row0, row0+1).
// ------------------------------------------------------------------------------------------------------------
template <int NT, bool XG, class Epi>
__device__ __forceinline__ void gemv_seg(Ctx& c, int seg, const float* x, int xstride, int ncols, Epi epi) {
  const uint32_t st = SMEM().seg[seg];
  const int gbeg = seg_begin(st), gn = seg_count(st);
  const float* xr[NT];
#pragma unroll
  for (int t = 0; t < NT; ++t) xr[t] = x + (size_t)(t < ncols ? t : 0) * xstride + c.lane * 4;
  for (int gi = 0; gi < gn; ++gi) {
    const Grp g = SMEM().grp[gbeg + gi];
    const int npairs = g.rows >> 1;
    const int m = g.m;
    float acc[4][NT];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int t = 0; t < NT; ++t) acc[a][t] = 0.f;
    for (int tl = 0; tl < g.ntiles; ++tl) {
      const int stage = (int)(c.tile_ctr % NS);
      const uint32_t par = (c.tile_ctr / NS) & 1u;
      mbar_wait(&SMEM().full[stage], par);
      const uint8_t* tile = SMEM().ring[stage];
      for (int j = 0; j < m; ++j) {
        const int kb = tl * m + j;
        float xv[NT][4];
#pragma unroll
        for (int t = 0; t < NT; ++t) {
          const float4* xp = reinterpret_cast<const float4*>(xr[t] + kb * 128);
          const float4 a = XG ? __ldcg(xp) : *xp;
          xv[t][0] = a.x; xv[t][1] = a.y; xv[t][2] = a.z; xv[t][3] = a.w;
        }
#pragma unroll
        for (int sl = 0; sl < 2; ++sl) {
          const int p = c.warp + NCW * sl;
          if (p < npairs) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int r = 2 * p + h;
              const uint4 w = *reinterpret_cast<const uint4*>(tile + ((size_t)(r * m + j) * 32 + c.lane) * 16);
              const float wf[4] = {__uint_as_float(w.x), __uint_as_float(w.y), __uint_as_float(w.z), __uint_as_float(w.w)};
#pragma unroll
              for (int t = 0; t < NT; ++t)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[sl * 2 + h][t] = fmaf(wf[e], xv[t][e], acc[sl * 2 + h][t]);
            }
          }
        }
      }
      __syncwarp();
      if (c.lane == 0) mbar_arrive(&SMEM().empty[stage]);
      c.tile_ctr++;
    }
#pragma unroll
    for (int sl = 0; sl < 2; ++sl) {
      const int p = c.warp + NCW * sl;
      if (p < npairs) {
        float v0[NT], v1[NT];
#pragma unroll
        for (int t = 0; t < NT; ++t) {
          float a = acc[sl * 2][t], b = acc[sl * 2 + 1][t];
#pragma unroll
          for (int o = 16; o; o >>= 1) {
            a += __shfl_xor_sync(0xffffffffu, a, o);
            b += __shfl_xor_sync(0xffffffffu, b, o);
          }
          v0[t] = a;
          v1[t] = b;
        }
        if (c.lane == 0) epi(g.row0 + 2 * p, v0, v1);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// Producer: stream the segments of the program in consumption order.
// ------------------------------------------------------------------------------------------------------------
// ---- split-key talker attention: which cached keys CTA split s of S handles, and how many 64-key ring tiles that is
constexpr int KVT_KEYS = 64;            // keys per ring tile: K rows at byte 0, V rows at byte KVT_VOFF (bf16, 256 B per row)
constexpr int KVT_VOFF = STAGE_BYTES / 2;
constexpr int PART_STRIDE = 132;
struct KvSlice { int j0, n, ntile; };
__device__ __forceinline__ KvSlice kv_slice(int nold, int S, int s) {
  int per = (nold + S - 1) / S;
  per = (per + 7) & ~7;
  const int j0 = min(s * per, nold), j1 = min(j0 + per, nold);
  return KvSlice{j0, j1 - j0, (j1 - j0 + KVT_KEYS - 1) / KVT_KEYS};
}

template <bool BF>
struct Producer {
  const KParams& P;
  Smem& s;
  uint32_t ctr = 0;     // tiles issued
  bool stopped = false;
  uint64_t pol_first;   // L2 eviction policy of the weight stream (evict_first)
  __device__ __forceinline__ explicit Producer(const KParams& p) : P(p), s(SMEM()) {
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol_first));
  }
  // tell the consumers' drain_producer() how many tiles were issued
  __device__ __forceinline__ void finish() {
    flag_st(&s.prod_issued, (int)ctr);
    __threadfence_block();
    flag_st(&s.prod_done, 1);
  }
  // segment sg, `rep` times over (the batched kernel replays a segment once per column block, see gemv_b)
  __device__ __forceinline__ void seg(int sg, int rep = 1) {
    if (stopped) return;
    const uint32_t st = s.seg[sg];
    const int gbeg = seg_begin(st), gn = seg_count(st);
    for (int r = 0; r < rep; ++r)
      for (int gi = 0; gi < gn; ++gi) {
        const Grp g = s.grp[gbeg + gi];
        const uint32_t bytes = tile_bytes(BF, g.rows, g.m);
        const uint8_t* src = P.tape + (size_t)g.off16 * 16;
        for (int tl = 0; tl < g.ntiles; ++tl) {
          const int stage = (int)(ctr % NS);
          const uint32_t par = ((ctr / NS) & 1u) ^ 1u;
          while (!mbar_try_wait(&s.empty[stage], par)) {
            if (flag_ld(&s.stop_flag)) {
              stopped = true;
              return;
            }
          }
          mbar_expect_tx(&s.full[stage], bytes);
          bulk_g2s_hint(s.ring[stage], src + (size_t)tl * bytes, bytes, &s.full[stage], pol_first);
          ++ctr;
        }
      }
  }
  // K/V rows of this CTA's key slice of layer l -> ring tiles (issued right behind the layer's QKV weights, so they
  // land while the QKV GEMV and its barrier are still in flight).  Must mirror attention_split().
  __device__ __forceinline__ void kv_tiles(const StackDev& S, int layer, int slot0, int kv_start) {
    if (stopped) return;
    const int Sx = P.attn_split, b = (int)blockIdx.x;
    if (b >= S.nH * Sx) return;
    const int h = b / Sx, sp = b - h * Sx, g = h / S.rep;
    const KvSlice sl = kv_slice(slot0 - kv_start, Sx, sp);
    for (int tl = 0; tl < sl.ntile; ++tl) {
      // a slice starts at a multiple of 8 keys, so a tile may straddle two pages: then it is two copies per matrix
      const int r0 = kv_start + sl.j0 + KVT_KEYS * tl;
      const int n = min(KVT_KEYS, sl.n - KVT_KEYS * tl), n1 = min(n, KV_PAGE - r0 % KV_PAGE);
      const uint32_t bytes = (uint32_t)n * 256u, b1 = (uint32_t)n1 * 256u;
      const int stage = (int)(ctr % NS);
      const uint32_t par = ((ctr / NS) & 1u) ^ 1u;
      while (!mbar_try_wait(&s.empty[stage], par)) {
        if (flag_ld(&s.stop_flag)) {
          stopped = true;
          return;
        }
      }
      mbar_expect_tx(&s.full[stage], 2 * bytes);
      bulk_g2s(s.ring[stage], kv_row(P.req.kv, S.L, S.nKV, 2, s.kvtab, 0, layer, g, r0), b1, &s.full[stage]);
      bulk_g2s(s.ring[stage] + KVT_VOFF, kv_row(P.req.kv, S.L, S.nKV, 2, s.kvtab, 1, layer, g, r0), b1,
               &s.full[stage]);
      if (n1 < n) {
        bulk_g2s(s.ring[stage] + b1, kv_row(P.req.kv, S.L, S.nKV, 2, s.kvtab, 0, layer, g, r0 + n1), bytes - b1,
                 &s.full[stage]);
        bulk_g2s(s.ring[stage] + KVT_VOFF + b1, kv_row(P.req.kv, S.L, S.nKV, 2, s.kvtab, 1, layer, g, r0 + n1),
                 bytes - b1, &s.full[stage]);
      }
      ++ctr;
    }
  }
  // kv_slot0 >= 0: talker step at cache slot kv_slot0 with split attention
  __device__ __forceinline__ void stack_layers(const StackDev& S, int rep = 1, int kv_slot0 = -1, int kv_start = 0) {
    for (int l = 0; l < S.L; ++l)
      for (int q = 0; q < 4; ++q) {
        seg(S.seg_base + 4 * l + q, rep);
        if (BF && q == 0 && kv_slot0 >= 0 && P.attn_split > 0 && kv_slot0 - kv_start >= ATTN_SPLIT_MIN)
          kv_tiles(S, l, kv_slot0, kv_start);
      }
  }
  // the code predictor's 15 passes: the MTP projection (pass 0), then per pass its layers and head.  rep0 / rep1: the
  // replays of pass 0's segments and of the 1-column segments (pass 0 carries two tokens per request)
  __device__ __forceinline__ void predictor(int rep0, int rep1) {
    for (int i = 0; i < P.ncb; ++i) {
      if (P.has_mtp && i == 0) seg(P.seg_mtp, rep0);
      stack_layers(P.p, i == 0 ? rep0 : rep1);
      seg(P.p.seg_head + i, rep1);
    }
  }
  // one frame of a fused launch, the order both decode kernels consume it in: the predictor, then the talker step at
  // cache slot kv_slot0 (-1: no split attention) and its head
  __device__ __forceinline__ void frame(int rep0, int rep1, int kv_slot0, int kv_start) {
    predictor(rep0, rep1);
    stack_layers(P.t, rep1, kv_slot0, kv_start);
    seg(P.t.seg_head, rep1);
  }
};

// ------------------------------------------------------------------------------------------------------------
// The new token's q-head h and the k and v rows of its kv group, out of its QKV row: warp 0 q, warp 1 k, warp 2 v; a
// lane owns e, e+32, e+64, e+96.  q and k get q_norm / k_norm and RoPE at rotary position rpos; the three rows go to
// qs / ks / vs.  append: this CTA also writes k and v to cache row `slot` (talker_graph StaticCache.update).  A split
// attention (attention_split) reads cached rows through the async proxy (TMA), in this launch or a later one, so every
// append is followed by a proxy fence.
// ------------------------------------------------------------------------------------------------------------
// XT: the QKV row is a tagged exchange (tag `tag`): the three rows are polled, not read after a grid barrier
template <bool BF, bool XT = false>
__device__ __forceinline__ void head_qkv(Ctx& c, const StackDev& S, int layer, int h, const float* qkv, int rpos,
                                         float* qs, float* ks, float* vs, void* kv, const int* pages, int slot,
                                         bool append, uint32_t tag = 0) {
  if (c.warp < 3) {
    const int what = c.warp, g = h / S.rep;
    const float* src = qkv + (what == 0 ? h * 128 : (what == 1 ? S.qd + g * 128 : S.qd + S.kd + g * 128));
    float v[4], nwv[4], cc[4], sv[4];
    {
      const int rp = rpos < 0 ? 0 : (rpos >= S.npos ? S.npos - 1 : rpos);
      const float* cs = S.cos + (size_t)rp * 128;
      const float* sn = S.sin + (size_t)rp * 128;
      const void* nw = what == 0 ? S.qnorm : S.knorm;
#pragma unroll
      for (int i = 0; i < 4; ++i) {  // all global loads of this step issued back to back
        const int e = c.lane + 32 * i;
        v[i] = XT ? __uint_as_float(ld_relaxed_u32(src + e)) : __ldcg(src + e);
        nwv[i] = what < 2 ? ldw<BF>(nw, (size_t)layer * 128 + e) : 0.f;
        cc[i] = what < 2 ? __ldg(cs + e) : 0.f;
        sv[i] = what < 2 ? __ldg(sn + e) : 0.f;
      }
      if constexpr (XT) {  // the loads above were the first poll: re-poll only the words still stale, then untag
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          uint32_t w = __float_as_uint(v[i]);
          if (!xtag_ok(w, tag)) w = xwait(c.P.xerr, src + c.lane + 32 * i, w, tag);
          v[i] = untag(w);
        }
      }
    }
    if (what < 2) {
      float ss = v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3];
#pragma unroll
      for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
      const float r = 1.0f / sqrtf(ss / 128.0f + S.eps);
#pragma unroll
      for (int i = 0; i < 4; ++i) v[i] = rnd<BF>(nwv[i] * rnd<BF>(v[i] * r));
      float o[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float rot = (i < 2) ? -v[i + 2] : v[i - 2];
        o[i] = rnd<BF>(rnd<BF>(v[i] * rnd<BF>(cc[i])) + rnd<BF>(rot * rnd<BF>(sv[i])));
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) v[i] = o[i];
    }
    float* dst = what == 0 ? qs : (what == 1 ? ks : vs);
#pragma unroll
    for (int i = 0; i < 4; ++i) dst[c.lane + 32 * i] = v[i];
    if (what > 0 && append) {
      uint8_t* cb = kv_row(kv, S.L, S.nKV, BF ? 2 : 4, pages, what - 1, layer, g, slot);
#pragma unroll
      for (int i = 0; i < 4; ++i) stw<BF>(cb, c.lane + 32 * i, v[i]);
      asm volatile("fence.proxy.async.global;" ::: "memory");
    }
  }
  csync();
}

// ------------------------------------------------------------------------------------------------------------
// Talker attention of one new token for one q-head over the KV cache (transformers eager_attention_forward semantics,
// GQA by repeat_kv): cache slot slot0, rotary position rpos0, keys from kv_start on.  qkv: the token's QKV row; pool /
// pages: the page pool and the request's page table; the head's output goes to att[h*128 .. h*128+128) in model dtype.
// Both kernels run it.
// ------------------------------------------------------------------------------------------------------------
template <bool BF, bool XT = false>
__device__ void attention_head(Ctx& c, const StackDev& S, int layer, int h, const float* __restrict__ qkv, void* pool,
                               const int* pages, void* att, int slot0, int rpos0, int kv_start, uint32_t tag = 0) {
  float* sc = SMEM().xs;            // scores [SEQMAX]
  float* qs = SMEM().xs + SEQMAX;   // [128]
  float* ks = qs + 128;             // [128]
  float* vs = ks + 128;             // [128]
  float* opart = vs + 128;          // [8][128]
  const int g = h / S.rep;
  const size_t esz = BF ? 2 : 4;
  // --- a. q/k norm + rope, v copy; the first q-head of each kv group appends the new row
  head_qkv<BF, XT>(c, S, layer, h, qkv, rpos0, qs, ks, vs, pool, pages, slot0, (h % S.rep) == 0, tag);
  const float scale = 0.08838834764831845f;  // 128^-0.5
  const int nk = slot0 + 1 - kv_start;       // visible keys
  const int nold = slot0 - kv_start;         // keys that live in the global cache
  // --- b. scores
  {
    constexpr int LPK = BF ? 16 : 32;  // lanes per key (16 bytes per lane)
    constexpr int KPW = 32 / LPK;      // keys per warp-instruction
    constexpr int EPL = BF ? 8 : 4;
    constexpr int U = 16;
    const int sub = c.lane % LPK, kin = c.lane / LPK;
    float q[EPL];
#pragma unroll
    for (int e = 0; e < EPL; ++e) q[e] = qs[sub * EPL + e];
    for (int base = 0; base < nold; base += NCW * KPW * U) {
      uint4 kv[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int jj = base + (u * NCW + c.warp) * KPW + kin;
        if (jj < nold)
          kv[u] = __ldcg(reinterpret_cast<const uint4*>(kv_row(pool, S.L, S.nKV, esz, pages, 0, layer, g, kv_start + jj)) + sub);
        else
          kv[u] = make_uint4(0, 0, 0, 0);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int jj = base + (u * NCW + c.warp) * KPW + kin;
        float d = 0.f;
        if constexpr (BF) {
          d = fmaf(q[0], bf_lo(kv[u].x), d); d = fmaf(q[1], bf_hi(kv[u].x), d);
          d = fmaf(q[2], bf_lo(kv[u].y), d); d = fmaf(q[3], bf_hi(kv[u].y), d);
          d = fmaf(q[4], bf_lo(kv[u].z), d); d = fmaf(q[5], bf_hi(kv[u].z), d);
          d = fmaf(q[6], bf_lo(kv[u].w), d); d = fmaf(q[7], bf_hi(kv[u].w), d);
        } else {
          d = fmaf(q[0], __uint_as_float(kv[u].x), d); d = fmaf(q[1], __uint_as_float(kv[u].y), d);
          d = fmaf(q[2], __uint_as_float(kv[u].z), d); d = fmaf(q[3], __uint_as_float(kv[u].w), d);
        }
#pragma unroll
        for (int o = LPK / 2; o; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
        if (sub == 0 && jj < nold) sc[jj] = rnd<BF>(rnd<BF>(d) * scale);
      }
    }
    if (c.warp == 0) {  // the new key (shared memory)
      float d = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) d = fmaf(qs[c.lane + 32 * i], ks[c.lane + 32 * i], d);
#pragma unroll
      for (int o = 16; o; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
      if (c.lane == 0) sc[nold] = rnd<BF>(rnd<BF>(d) * scale);
    }
  }
  csync();
  // --- c. softmax (fp32, then rounded to dtype like softmax(..., dtype=float32).to(q.dtype))
  float mx = -INFINITY;
  for (int j = c.tid; j < nk; j += NCT) mx = fmaxf(mx, sc[j]);
  mx = block_max(c, mx);
  float sm = 0.f;
  for (int j = c.tid; j < nk; j += NCT) {
    const float e = expf(sc[j] - mx);
    sc[j] = e;
    sm += e;
  }
  sm = block_sum(c, sm);
  for (int j = c.tid; j < nk; j += NCT) sc[j] = rnd<BF>(sc[j] / sm);
  csync();
  // --- d. P.V : 16-byte loads; bf16: 16 lanes per key (lane owns 8 dims), 2 keys per warp instruction
  {
    constexpr int LPK = BF ? 16 : 32;
    constexpr int KPW = 32 / LPK;
    constexpr int EPL = BF ? 8 : 4;
    constexpr int U = 16;
    const int sub = c.lane % LPK, kin = c.lane / LPK;
    float acc[EPL];
#pragma unroll
    for (int e = 0; e < EPL; ++e) acc[e] = 0.f;
    for (int base = 0; base < nold; base += NCW * KPW * U) {
      uint4 vv[U];
      float pv[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int jj = base + (u * NCW + c.warp) * KPW + kin;
        if (jj < nold) {
          vv[u] = __ldcg(reinterpret_cast<const uint4*>(kv_row(pool, S.L, S.nKV, esz, pages, 1, layer, g, kv_start + jj)) + sub);
          pv[u] = sc[jj];
        } else {
          vv[u] = make_uint4(0, 0, 0, 0);
          pv[u] = 0.f;
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if constexpr (BF) {
          acc[0] = fmaf(pv[u], bf_lo(vv[u].x), acc[0]); acc[1] = fmaf(pv[u], bf_hi(vv[u].x), acc[1]);
          acc[2] = fmaf(pv[u], bf_lo(vv[u].y), acc[2]); acc[3] = fmaf(pv[u], bf_hi(vv[u].y), acc[3]);
          acc[4] = fmaf(pv[u], bf_lo(vv[u].z), acc[4]); acc[5] = fmaf(pv[u], bf_hi(vv[u].z), acc[5]);
          acc[6] = fmaf(pv[u], bf_lo(vv[u].w), acc[6]); acc[7] = fmaf(pv[u], bf_hi(vv[u].w), acc[7]);
        } else {
          acc[0] = fmaf(pv[u], __uint_as_float(vv[u].x), acc[0]); acc[1] = fmaf(pv[u], __uint_as_float(vv[u].y), acc[1]);
          acc[2] = fmaf(pv[u], __uint_as_float(vv[u].z), acc[2]); acc[3] = fmaf(pv[u], __uint_as_float(vv[u].w), acc[3]);
        }
      }
    }
    if constexpr (BF) {  // fold the two key halves of the warp: lanes sub and sub+16 own the same dims
#pragma unroll
      for (int e = 0; e < EPL; ++e) acc[e] += __shfl_xor_sync(0xffffffffu, acc[e], 16);
    }
    if (c.warp == 0 && kin == 0) {
      const float pj = sc[nold];
#pragma unroll
      for (int e = 0; e < EPL; ++e) acc[e] = fmaf(pj, vs[sub * EPL + e], acc[e]);
    }
    if (kin == 0) {
      float* op = opart + c.warp * 128 + sub * EPL;
#pragma unroll
      for (int e = 0; e < EPL; ++e) op[e] = acc[e];
    }
  }
  csync();
  if (c.tid < 128) {
    float o = 0.f;
#pragma unroll
    for (int w = 0; w < NCW; ++w) o += opart[w * 128 + c.tid];
    stw<BF>(att, (size_t)h * 128 + c.tid, o);
  }
  csync();
}

// ------------------------------------------------------------------------------------------------------------
// Talker attention with the keys of every q-head split over P.attn_split CTAs (bf16 engines, one token).
// CTA b = h * S + s handles q-head h and the s-th slice of the cached keys; the K/V rows of that slice were staged
// into ring tiles by the producer warp (TMA bulk copies issued behind the QKV weights, i.e. before the barrier that
// precedes this function), so scores and P.V run out of shared memory.  Each CTA publishes an un-normalised partial
// (sum_j e^{s_j - m} v_j, m, sum_j e^{s_j - m}); the CTA that arrives last at the head's counter merges the S
// partials in split order -- deterministic whichever CTA that is -- and writes the head's slice of ATT.
// Differences to attention_head(): probabilities are not rounded to bf16 before P.V (higher precision, not lower).
// ------------------------------------------------------------------------------------------------------------
template <bool BF>
__device__ void attention_split(Ctx& c, const StackDev& S, int layer, int slot0, int rpos0, int kv_start) {
  const KParams& P = c.P;
  const int Sx = P.attn_split, b = (int)blockIdx.x;
  if (b >= S.nH * Sx) return;  // spare CTAs
  const int h = b / Sx, sp = b - h * Sx;
  float* sc = SMEM().xs;           // scores / exponentials of this slice (+ the new key)
  float* qs = SMEM().xs + 512;     // [128]
  float* ks = qs + 128;            // [128]
  float* vs = ks + 128;            // [128]
  float* opart = vs + 128;         // [8][128]
  // --- a. q/k norm + rope, v copy; one CTA per kv group appends the new row
  head_qkv<BF, BF>(c, S, layer, h, P.QKV, rpos0, qs, ks, vs, P.req.kv, SMEM().kvtab, slot0, sp == 0 && (h % S.rep) == 0,
                   c.xtag);
  const KvSlice sl = kv_slice(slot0 - kv_start, Sx, sp);
  const bool has_new = sp == Sx - 1;
  const int nloc = sl.n + (has_new ? 1 : 0);
  const float scale = 0.08838834764831845f;  // 128^-0.5
  const int sub = c.lane & 15, kin = c.lane >> 4;  // 16 lanes per key (16 bytes each), 2 keys per warp instruction
  // --- b. scores out of the staged K rows
  {
    float q[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) q[e] = qs[sub * 8 + e];
    for (int tl = 0; tl < sl.ntile; ++tl) {
      const uint32_t tc = c.tile_ctr + (uint32_t)tl;
      const int stage = (int)(tc % NS);
      mbar_wait(&SMEM().full[stage], (tc / NS) & 1u);
      const uint8_t* kt = SMEM().ring[stage];
      const int n = min(KVT_KEYS, sl.n - KVT_KEYS * tl);
      for (int j0 = 0; j0 < n; j0 += 2 * NCW) {
        const int jj = j0 + c.warp * 2 + kin;
        float d = 0.f;
        if (jj < n) {
          const uint4 kv = *reinterpret_cast<const uint4*>(kt + (size_t)jj * 256 + sub * 16);
          d = fmaf(q[0], bf_lo(kv.x), d); d = fmaf(q[1], bf_hi(kv.x), d);
          d = fmaf(q[2], bf_lo(kv.y), d); d = fmaf(q[3], bf_hi(kv.y), d);
          d = fmaf(q[4], bf_lo(kv.z), d); d = fmaf(q[5], bf_hi(kv.z), d);
          d = fmaf(q[6], bf_lo(kv.w), d); d = fmaf(q[7], bf_hi(kv.w), d);
        }
#pragma unroll
        for (int o = 8; o; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
        if (sub == 0 && jj < n) sc[KVT_KEYS * tl + jj] = rnd<BF>(rnd<BF>(d) * scale);
      }
    }
    if (has_new && c.warp == 0) {
      float d = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) d = fmaf(qs[c.lane + 32 * i], ks[c.lane + 32 * i], d);
#pragma unroll
      for (int o = 16; o; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
      if (c.lane == 0) sc[sl.n] = rnd<BF>(rnd<BF>(d) * scale);
    }
  }
  csync();
  // --- c. slice-local softmax statistics (fp32)
  float mx = -INFINITY;
  for (int j = c.tid; j < nloc; j += NCT) mx = fmaxf(mx, sc[j]);
  mx = block_max(c, mx);
  float sm = 0.f;
  for (int j = c.tid; j < nloc; j += NCT) {
    const float e = expf(sc[j] - mx);
    sc[j] = e;
    sm += e;
  }
  sm = block_sum(c, sm);
  // --- d. un-normalised P.V out of the staged V rows
  {
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    for (int tl = 0; tl < sl.ntile; ++tl) {
      const uint32_t tc = c.tile_ctr + (uint32_t)tl;
      const uint8_t* vt = SMEM().ring[(int)(tc % NS)] + KVT_VOFF;
      const int n = min(KVT_KEYS, sl.n - KVT_KEYS * tl);
      for (int j0 = 0; j0 < n; j0 += 2 * NCW) {
        const int jj = j0 + c.warp * 2 + kin;
        if (jj < n) {
          const float pv = sc[KVT_KEYS * tl + jj];
          const uint4 vv = *reinterpret_cast<const uint4*>(vt + (size_t)jj * 256 + sub * 16);
          acc[0] = fmaf(pv, bf_lo(vv.x), acc[0]); acc[1] = fmaf(pv, bf_hi(vv.x), acc[1]);
          acc[2] = fmaf(pv, bf_lo(vv.y), acc[2]); acc[3] = fmaf(pv, bf_hi(vv.y), acc[3]);
          acc[4] = fmaf(pv, bf_lo(vv.z), acc[4]); acc[5] = fmaf(pv, bf_hi(vv.z), acc[5]);
          acc[6] = fmaf(pv, bf_lo(vv.w), acc[6]); acc[7] = fmaf(pv, bf_hi(vv.w), acc[7]);
        }
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] += __shfl_xor_sync(0xffffffffu, acc[e], 16);  // fold the two keys of a warp instruction
    if (has_new && c.warp == 0 && kin == 0) {
      const float pj = sc[sl.n];
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] = fmaf(pj, vs[sub * 8 + e], acc[e]);
    }
    if (kin == 0) {
#pragma unroll
      for (int e = 0; e < 8; ++e) opart[c.warp * 128 + sub * 8 + e] = acc[e];
    }
    // hand the ring tiles back to the producer
    __syncwarp();
    if (c.lane == 0)
      for (int tl = 0; tl < sl.ntile; ++tl) mbar_arrive(&SMEM().empty[(int)((c.tile_ctr + (uint32_t)tl) % NS)]);
    c.tile_ctr += (uint32_t)sl.ntile;
  }
  csync();
  float* part = P.PART + ((size_t)h * Sx + sp) * PART_STRIDE;
  if (c.tid < 128) {
    float o = 0.f;
#pragma unroll
    for (int w = 0; w < NCW; ++w) o += opart[w * 128 + c.tid];
    part[c.tid] = o;
  }
  if (c.tid == 128) { part[128] = mx; part[129] = sm; }
  // --- e. arrive at the head's counter; the last split merges
  csync();
  if (c.tid == 0) {
    unsigned old;
    asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(P.attn_cnt + h), "r"(1u) : "memory");
    SMEM().ibc[0] = ((old + 1u) % (unsigned)Sx) == 0u ? 1 : 0;
  }
  csync();
  if (SMEM().ibc[0] && c.tid < 128) {
    const float* ph = P.PART + (size_t)h * Sx * PART_STRIDE;
    float M = -INFINITY;
    for (int s2 = 0; s2 < Sx; ++s2) M = fmaxf(M, __ldcg(ph + (size_t)s2 * PART_STRIDE + 128));
    float L = 0.f, o = 0.f;
    for (int s2 = 0; s2 < Sx; ++s2) {
      const float m2 = __ldcg(ph + (size_t)s2 * PART_STRIDE + 128);
      const float w = m2 == -INFINITY ? 0.f : expf(m2 - M);
      L = fmaf(w, __ldcg(ph + (size_t)s2 * PART_STRIDE + 129), L);
      o = fmaf(w, __ldcg(ph + (size_t)s2 * PART_STRIDE + c.tid), o);
    }
    stw<BF>(P.ATT, (size_t)h * 128 + c.tid, o / L);
  }
  csync();
}

// ------------------------------------------------------------------------------------------------------------
// Sampling (sampling.py:32-66 + :10-29), computed redundantly and deterministically by every CTA.
// Returns the token to all consumer threads.
// ------------------------------------------------------------------------------------------------------------
struct SampleArgs {
  const float* logits;  // global fp32 (dtype-rounded values)
  int V;
  Sampling sp;
  float u;
  bool use_penalty;     // repetition penalty over the seen bitmap
  int sup0;             // ids in [sup0, V) except eos are suppressed (V = none)   generate.py:46-50
  bool suppress_eos;
  int eos;
  float* lp = nullptr;  // when set, thread 0 writes the log-probability of the drawn id here (DESIGN.md §4)
  uint32_t xtag = 0;    // nonzero (bf16): logits is a tagged exchange with this tag, polled instead of read after a barrier
};

__device__ __forceinline__ uint32_t fkey(float f) {  // order-preserving float -> uint
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float fkey_inv(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

template <bool BF>
__device__ int sample_block(Ctx& c, const SampleArgs& a) {
  float* lg = SMEM().xs;  // [V]
  const int V = a.V;
  const int sup0 = a.sup0;
  if (BF && a.xtag) {  // every word of the thread's share in flight at once, then only the stale ones re-polled
    constexpr int VPT = VMAX / NCT;
    uint32_t w[VPT];
#pragma unroll
    for (int i = 0; i < VPT; ++i) w[i] = c.tid + i * NCT < V ? ld_relaxed_u32(a.logits + c.tid + i * NCT) : a.xtag;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      if (!xtag_ok(w[i], a.xtag)) w[i] = xwait(c.P.xerr, a.logits + c.tid + i * NCT, w[i], a.xtag);
      if (c.tid + i * NCT < V) lg[c.tid + i * NCT] = untag(w[i]);
    }
  }
  for (int v = c.tid; v < V; v += NCT) {
    float l = (BF && a.xtag) ? lg[v] : __ldcg(a.logits + v);
    if (a.use_penalty && a.sp.penalty != 1.0f && ((SMEM().seen[v >> 5] >> (v & 31)) & 1u))
      l = l > 0.f ? rnd<BF>(l / a.sp.penalty) : rnd<BF>(l * a.sp.penalty);
    if ((v >= sup0 && v != a.eos) || (a.suppress_eos && v == a.eos)) l = -INFINITY;
    lg[v] = l;
  }
  csync();
  if (!a.sp.do_sample) {  // argmax, lowest index among maxima
    float bm = -INFINITY;
    int bi = 0x7fffffff;
    for (int v = c.tid; v < V; v += NCT) {
      const float l = lg[v];
      if (l > bm || (l == bm && v < bi)) { bm = l; bi = v; }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, bm, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (om > bm || (om == bm && oi < bi)) { bm = om; bi = oi; }
    }
    if (c.lane == 0) { SMEM().red[c.warp] = bm; SMEM().hist[c.warp] = bi; }
    csync();
    float m = SMEM().red[0];
    int bi2 = SMEM().hist[0];
    for (int w = 1; w < NCW; ++w) {
      const float om = SMEM().red[w];
      const int oi = SMEM().hist[w];
      if (om > m || (om == m && oi < bi2)) { m = om; bi2 = oi; }
    }
    if (a.lp) {  // log-softmax at the argmax, no temperature: (l_tok - m) - log(sum exp(l - m)) with l_tok == m
      csync();   // every warp has read red[] / hist[] above before block_sum overwrites red[]
      float se = 0.f;
      for (int v = c.tid; v < V; v += NCT) se += expf(lg[v] - m);
      se = block_sum(c, se);
      if (c.tid == 0) *a.lp = -logf(se);
    }
    csync();
    return bi2;
  }
  // temperature
  for (int v = c.tid; v < V; v += NCT) lg[v] = rnd<BF>(lg[v] / a.sp.temperature);
  csync();
  // top-k with ties kept: threshold = k-th largest value (sampling.py:54-56)
  if (a.sp.top_k > 0 && a.sp.top_k < V) {
    uint32_t prefix = 0, mask = 0;
    int remaining = a.sp.top_k;
    for (int pass = 0; pass < (BF ? 2 : 4); ++pass) {  // bf16-rounded logits have 16 zero low bits
      const int shift = 24 - 8 * pass;
      SMEM().hist[c.tid] = 0;
      csync();
      for (int v = c.tid; v < V; v += NCT) {
        const uint32_t k = fkey(lg[v]);
        if ((k & mask) == prefix) atomicAdd(&SMEM().hist[(k >> shift) & 255u], 1);
      }
      csync();
      if (c.warp == 0) {  // lane L owns bins 255-8L .. 248-8L (descending)
        int cnt[8], tot = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) { cnt[i] = SMEM().hist[255 - 8 * c.lane - i]; tot += cnt[i]; }
        int incl = tot;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int n = __shfl_up_sync(0xffffffffu, incl, o);
          if (c.lane >= o) incl += n;
        }
        const int excl = incl - tot;
        if (excl < remaining && incl >= remaining) {
          int run = excl;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            if (run < remaining && run + cnt[i] >= remaining) {
              SMEM().ibc[0] = 255 - 8 * c.lane - i;
              SMEM().ibc[1] = remaining - run;
            }
            run += cnt[i];
          }
        }
      }
      csync();
      prefix |= ((uint32_t)SMEM().ibc[0]) << shift;
      mask |= 255u << shift;
      remaining = SMEM().ibc[1];
      csync();
    }
    const float kth = fkey_inv(prefix);
    for (int v = c.tid; v < V; v += NCT)
      if (lg[v] < kth) lg[v] = -INFINITY;
    csync();
  }
  // top-p (fp32 semantics, order: value desc then index asc; keep position 0 and every position with cum <= top_p)
  if (a.sp.top_p < 1.0f) {
    float* sl = &SMEM().xin[0][0];                                      // sorted values [V] (xin is free here)
    uint16_t* rk = reinterpret_cast<uint16_t*>(SMEM().xs + VMAX);       // ranks [V]
    for (int v = c.tid; v < V; v += NCT) {
      const float l = lg[v];
      int r = 0;
      for (int w = 0; w < V; ++w) {
        const float o = lg[w];
        r += (o > l || (o == l && w < v)) ? 1 : 0;
      }
      rk[v] = (uint16_t)r;
      sl[r] = l;
    }
    csync();
    if (c.tid == 0) {
      const float m0 = sl[0];
      float S = 0.f;
      for (int i = 0; i < V; ++i) S += expf(sl[i] - m0);
      float cum = 0.f;
      int keep = 1;
      for (int i = 0; i < V; ++i) {
        cum += expf(sl[i] - m0) / S;
        if (i > 0 && !(cum > a.sp.top_p)) keep = i + 1;
        if (cum > a.sp.top_p && i > 0) break;
      }
      SMEM().ibc[2] = keep;
    }
    csync();
    const int keep = SMEM().ibc[2];
    for (int v = c.tid; v < V; v += NCT)
      if ((int)rk[v] >= keep) lg[v] = -INFINITY;
    csync();
  }
  // the processed row the draw uses, kept for the log-probability (the softmax below overwrites lg; xin is free here)
  float* lraw = &SMEM().xin[0][0];
  if (a.lp)
    for (int v = c.tid; v < V; v += NCT) lraw[v] = lg[v];
  // softmax -> probabilities in model dtype (F.softmax on a dtype tensor)
  float mx = -INFINITY;
  for (int v = c.tid; v < V; v += NCT) mx = fmaxf(mx, lg[v]);
  mx = block_max(c, mx);
  float sm = 0.f;
  for (int v = c.tid; v < V; v += NCT) {
    const float e = expf(lg[v] - mx);
    lg[v] = e;
    sm += e;
  }
  sm = block_sum(c, sm);
  for (int v = c.tid; v < V; v += NCT) lg[v] = rnd<BF>(lg[v] / sm);
  csync();
  // inverse-CDF draw, summation order fixed (oracle/qwen3_tts_oracle.py draw_inverse_cdf)
  const int CH = (V + NCT - 1) / NCT;
  float cs = 0.f;
  for (int j = 0; j < CH; ++j) {
    const int idx = c.tid * CH + j;
    if (idx < V) cs += lg[idx];
  }
  float incl = cs;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float n = __shfl_up_sync(0xffffffffu, incl, o);
    if (c.lane >= o) incl += n;
  }
  if (c.lane == 31) SMEM().red[c.warp] = incl;
  if (c.tid == 0) {
    SMEM().ibc[3] = -1;
    SMEM().ibc[0] = 0x7fffffff;
  }
  csync();
  float woff = 0.f, total = 0.f;
  for (int w = 0; w < NCW; ++w) {
    if (w == c.warp) woff = total;
    total += SMEM().red[w];
  }
  incl += woff;
  const float target = a.u * total;
  float excl = __shfl_up_sync(0xffffffffu, incl, 1);
  if (c.lane == 0) excl = woff;
  // lowest chunk whose inclusive prefix exceeds the target (prefix sums need not be monotone in fp32; the
  // oracle takes the first such chunk too)
  const bool hit = incl > target;
  if (hit) atomicMin(&SMEM().ibc[0], c.tid);
  csync();
  if (hit && SMEM().ibc[0] == c.tid) {
    float run = excl;
    int pick = -1;
    for (int j = 0; j < CH; ++j) {
      const int idx = c.tid * CH + j;
      if (idx >= V) break;
      run += lg[idx];
      if (run > target && lg[idx] > 0.f) { pick = idx; break; }
    }
    SMEM().ibc[3] = pick;
  }
  csync();
  int tok = SMEM().ibc[3];
  if (tok < 0) {  // rounding left nothing selected: last index with p > 0
    int best = -1;
    for (int v = c.tid; v < V; v += NCT)
      if (lg[v] > 0.f) best = v > best ? v : best;
#pragma unroll
    for (int o = 16; o; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    if (c.lane == 0) SMEM().hist[c.warp] = best;
    csync();
    tok = SMEM().hist[0];
    for (int w = 1; w < NCW; ++w) tok = max(tok, SMEM().hist[w]);
    if (tok < 0) tok = 0;
  }
  // fp32 log-softmax of the processed row at the drawn id, from the max and exp-sum the softmax reduced
  if (a.lp && c.tid == 0) *a.lp = (lraw[tok] - mx) - logf(sm);
  csync();
  return tok;
}

// ------------------------------------------------------------------------------------------------------------
// Tensor-core GEMV (bf16): the tape holds mma.sync m16n8k16 A-fragments in register order, so one LDS.128 per lane
// feeds one mma (16 rows x 16 k).  The activation vector(s) x (bf16, token t at x + t * ldx) enter as the B operand
// (column n = token; for 8-row "HALF" tiles columns 2n / 2n+1 carry the two K halves, rows 0-7 / 8-15 of the tile
// hold the matching halves of the weight rows, and c0 + c3 is the full dot product).  Warps split the k-groups of a
// tile; partial accumulators are combined in shared memory in a fixed order.  x is the staging vector in shared memory
// or (XG) an L2-resident vector in global memory; XG loads a warp's B fragments one ring tile ahead, so that the L2
// round trip overlaps the previous tile's MMAs (a tile holds at most 16 k-groups, two per warp).
//   pre(row, tok) -> float   value fetched BEFORE streaming starts (residual), handed back to epi
//   epi(row, tok, v, vup, aux)   GU tiles: row = pair index, v = gate, vup = up
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mma_bf16(float* d, const uint4& a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w), "r"(b0), "r"(b1));
}

template <int NT, bool XG, class Pre, class Epi>
__device__ __forceinline__ void gemv_mma(Ctx& c, int seg, int K, const __nv_bfloat16* x, int ldx, Pre pre, Epi epi) {
  float* red = SMEM().xs + XS_FLOATS / 2;  // [NCW][2][4][32] partial accumulators
  const uint32_t st = SMEM().seg[seg];
  const int gbeg = seg_begin(st), gn = seg_count(st);
  const int gq = c.lane >> 2, t = c.lane & 3;
  for (int gi = 0; gi < gn; ++gi) {
    const Grp g = SMEM().grp[gbeg + gi];
    const int n_mt = grp_nmt(g.rows), kind = grp_kind(g.rows), G = g.m;
    int tok, koff;
    bool bvalid;
    if (kind == 1) { tok = gq >> 1; koff = (gq & 1) * (K >> 1); bvalid = gq < 2 * NT; }
    else { tok = gq; koff = 0; bvalid = gq < NT; }
    const __nv_bfloat16* xb = x + (bvalid ? tok * ldx + koff : 0) + 16 * t;
    uint4 bn[2][2];   // XG: B fragments of the next tile, k-groups qq = warp and warp + NCW
    auto fetch_b = [&](int tl) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int qq = c.warp + NCW * i, kg = tl * G + qq;
        bn[i][0] = make_uint4(0, 0, 0, 0); bn[i][1] = make_uint4(0, 0, 0, 0);
        if (bvalid && qq < G) {
          bn[i][0] = __ldcg(reinterpret_cast<const uint4*>(xb + 64 * kg));
          bn[i][1] = __ldcg(reinterpret_cast<const uint4*>(xb + 64 * kg + 8));
        }
      }
    };
    if constexpr (XG) fetch_b(0);
    float aux[4] = {0.f, 0.f, 0.f, 0.f};
    if (c.warp < n_mt) {
      if (kind == 0) {
        const int rA = g.row0 + c.warp * 16 + gq;
        if (2 * t < NT) { aux[0] = pre(rA, 2 * t); aux[2] = pre(rA + 8, 2 * t); }
        if (2 * t + 1 < NT) { aux[1] = pre(rA, 2 * t + 1); aux[3] = pre(rA + 8, 2 * t + 1); }
      } else if (kind == 1) {
        if (t < NT) aux[0] = pre(g.row0 + gq, t);
      }
    }
    float acc[2][4];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[a][r] = 0.f;
    for (int tl = 0; tl < g.ntiles; ++tl) {
      uint4 bc[2][2];
      if constexpr (XG) {
#pragma unroll
        for (int i = 0; i < 2; ++i) { bc[i][0] = bn[i][0]; bc[i][1] = bn[i][1]; }
        if (tl + 1 < g.ntiles) fetch_b(tl + 1);
      }
      const int stage = (int)(c.tile_ctr % NS);
      const uint32_t par = (c.tile_ctr / NS) & 1u;
      mbar_wait(&SMEM().full[stage], par);
      const uint8_t* tile = SMEM().ring[stage];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int qq = c.warp + NCW * i;
        if (qq >= G) break;
        const int kg = tl * G + qq;
        uint4 blo = make_uint4(0, 0, 0, 0), bhi = make_uint4(0, 0, 0, 0);
        if constexpr (XG) {
          blo = bc[i][0];
          bhi = bc[i][1];
        } else if (bvalid) {
          blo = *reinterpret_cast<const uint4*>(xb + 64 * kg);
          bhi = *reinterpret_cast<const uint4*>(xb + 64 * kg + 8);
        }
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          if (mt < n_mt) {
            const uint4* A = reinterpret_cast<const uint4*>(tile + ((size_t)(mt * G + qq) * 4) * 512) + c.lane;
            const uint4 a0 = A[0], a1 = A[32], a2 = A[64], a3 = A[96];
            mma_bf16(acc[mt], a0, blo.x, blo.y);
            mma_bf16(acc[mt], a1, blo.z, blo.w);
            mma_bf16(acc[mt], a2, bhi.x, bhi.y);
            mma_bf16(acc[mt], a3, bhi.z, bhi.w);
          }
        }
      }
      __syncwarp();
      if (c.lane == 0) mbar_arrive(&SMEM().empty[stage]);
      c.tile_ctr++;
    }
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
      if (mt < n_mt)
#pragma unroll
        for (int r = 0; r < 4; ++r) red[((c.warp * 2 + mt) * 4 + r) * 32 + c.lane] = acc[mt][r];
    csync();
    if (c.warp < n_mt) {
      const int mt = c.warp;
      float cv[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        float sm = 0.f;
#pragma unroll
        for (int w = 0; w < NCW; ++w) sm += red[((w * 2 + mt) * 4 + r) * 32 + c.lane];
        cv[r] = sm;
      }
      if (kind == 2) {
        const int pair = g.row0 + mt * 8 + gq;
        if (2 * t < NT) epi(pair, 2 * t, cv[0], cv[2], 0.f);
        if (2 * t + 1 < NT) epi(pair, 2 * t + 1, cv[1], cv[3], 0.f);
      } else if (kind == 0) {
        const int rA = g.row0 + mt * 16 + gq;
        if (2 * t < NT) { epi(rA, 2 * t, cv[0], 0.f, aux[0]); epi(rA + 8, 2 * t, cv[2], 0.f, aux[2]); }
        if (2 * t + 1 < NT) { epi(rA, 2 * t + 1, cv[1], 0.f, aux[1]); epi(rA + 8, 2 * t + 1, cv[3], 0.f, aux[3]); }
      } else {
        if (t < NT) epi(g.row0 + gq, t, cv[0] + cv[3], 0.f, aux[0]);
      }
    }
    csync();
  }
}

// dispatch: bf16 -> tensor-core path, fp32 -> FMA path.  The input is the staging vector (K per token) or, XG, the
// model-dtype vectors xg [nt][ldx] in global memory, read in place
template <bool BF, bool GU, bool XG = false, class Pre, class Epi>
__device__ __forceinline__ void gemv_any(Ctx& c, int seg, int nt, int K, Pre pre, Epi epi, const void* xg = nullptr,
                                         int ldx = 0) {
  if constexpr (BF) {
    const __nv_bfloat16* x = XG ? reinterpret_cast<const __nv_bfloat16*>(xg) : reinterpret_cast<const __nv_bfloat16*>(SMEM().xs);
    const int ld = XG ? ldx : K;
    if (nt == 1) gemv_mma<1, XG>(c, seg, K, x, ld, pre, epi);
    else gemv_mma<2, XG>(c, seg, K, x, ld, pre, epi);
  } else {
    auto epi2 = [&](int row0, const float* v0, const float* v1) {
      for (int t = 0; t < nt; ++t) {
        if constexpr (GU) {
          epi(row0 >> 1, t, v0[t], v1[t], 0.f);
        } else {
          epi(row0, t, v0[t], 0.f, pre(row0, t));
          epi(row0 + 1, t, v1[t], 0.f, pre(row0 + 1, t));
        }
      }
    };
    const float* x = XG ? reinterpret_cast<const float*>(xg) : SMEM().xs;
    const int ld = XG ? ldx : K;
    if (nt == 1) gemv_seg<1, XG>(c, seg, x, ld, 1, epi2);
    else gemv_seg<2, XG>(c, seg, x, ld, 2, epi2);
  }
}

// staging vector element store: bf16 array (tensor-core path) or fp32 array (fp32 parity mode), both in s.xs
template <bool BF>
__device__ __forceinline__ void xs_put(Ctx& c, int idx, float v) {
  if constexpr (BF) reinterpret_cast<__nv_bfloat16*>(SMEM().xs)[idx] = __float2bfloat16_rn(v);
  else SMEM().xs[idx] = v;
}
template <bool BF>
__device__ __forceinline__ float xs_get(Ctx& c, int idx) {
  if constexpr (BF) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(SMEM().xs)[idx]);
  else return SMEM().xs[idx];
}

// ------------------------------------------------------------------------------------------------------------
// Predictor-size attention (cache <= 32 slots, i.e. <= 17 keys) of one request, all heads: one warp per kv group; a
// lane owns dims [4*lane, 4*lane+4) of every 128-vector.  The single-sequence kernel runs it redundantly in EVERY CTA
// and writes the result straight into the staging vector that feeds o_proj (no attention exchange, one grid barrier
// less per layer; CTA 0 appends the new K/V).  The batched kernel runs it in one CTA per request, which appends.
// ------------------------------------------------------------------------------------------------------------
// NT == 2 is the predictor prefill (slot0 == 0: no cached keys at all); NT == 1 the single-token passes.
// Register budget is 168/thread (9 warps per SM), so K rows and V rows are fetched in two round trips.
// ------------------------------------------------------------------------------------------------------------
// Warp reduce-scatter of 34 per-lane partial sums (2 heads x 17 keys of the predictor attention): instead of a 5-round
// butterfly on every value (170 shuffles, every lane ends with every sum), each round halves the value set -- a lane
// keeps one half and hands the other to its partner -- so 36 shuffles leave every sum on exactly one lane.  The owner's
// value is bit-identical to the butterfly's (same pairing tree, fp32 addition commutes).  own_lane / own_slot: where
// the sum of original index idx ends up.
// ------------------------------------------------------------------------------------------------------------
template <int N, int O>
__device__ __forceinline__ void rs_step(float* a, int lane) {
  constexpr int HH = (N + 1) / 2;
  const bool up = (lane & O) != 0;
#pragma unroll
  for (int i = 0; i < HH; ++i) {
    const float lo = a[i];
    const float hi = (i + HH < N) ? a[i + HH] : 0.f;
    const float send = up ? lo : hi, keep = up ? hi : lo;
    a[i] = keep + __shfl_xor_sync(0xffffffffu, send, O);
  }
}
__host__ __device__ constexpr int rs34_lane(int idx) {
  int l = 0, r = idx;
  if (r >= 17) { l |= 16; r -= 17; }
  if (r >= 9) { l |= 8; r -= 9; }
  if (r >= 5) { l |= 4; r -= 5; }
  if (r >= 3) { l |= 2; r -= 3; }
  if (r >= 2) { l |= 1; r -= 2; }
  return l;
}
__host__ __device__ constexpr int rs34_slot(int idx) {
  int r = idx;
  if (r >= 17) r -= 17;
  if (r >= 9) r -= 9;
  if (r >= 5) r -= 5;
  if (r >= 3) r -= 3;
  if (r >= 2) r -= 2;
  return r;
}
// scores sc[2][1][17] (per-lane partials) -> mine[hh] = the full dot product of key `lane` (lanes >= 17: untouched)
template <int HHI = 0, int J = 0>
__device__ __forceinline__ void rs34_gather(const float* a, int lane, float* mine) {
  if constexpr (HHI < 2) {
    constexpr int idx = HHI * 17 + J;
    const float v = __shfl_sync(0xffffffffu, a[rs34_slot(idx)], rs34_lane(idx));
    if (lane == J) mine[HHI] = v;
    if constexpr (J + 1 < 17) rs34_gather<HHI, J + 1>(a, lane, mine);
    else rs34_gather<HHI + 1, 0>(a, lane, mine);
  }
}

template <bool BF>
struct SmallKV {  // what a one-token pass of the attention reads besides its QKV row, fetched in the shadow of the QKV
                  // barrier: cached K/V rows of this warp's kv group and (bf16) the layer's q/k norm weights and the
                  // RoPE row.  The fp32 parity kernel loads the latter in the attention: preloading them raised its spills.
  using Raw = typename std::conditional<BF, uint2, float4>::type;
  Raw k[16], v[16];
  float4 qn, kn, cs, sn;   // dims [4 * lane, 4 * lane + 4)
};
// loads of the q/k norm weights and of the RoPE row of position rp (clamped to the table): attention_small_all issues
// them itself when nothing was preloaded
template <bool BF>
__device__ __forceinline__ void small_norm_rope_load(Ctx& c, const StackDev& S, int layer, int rp, float4& qn4,
                                                     float4& kn4, float4& cs4, float4& sn4) {
  const int L4 = 4 * c.lane;
  float qn[4], kn[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    qn[i] = ldw<BF>(S.qnorm, (size_t)layer * 128 + L4 + i);
    kn[i] = ldw<BF>(S.knorm, (size_t)layer * 128 + L4 + i);
  }
  qn4 = make_float4(qn[0], qn[1], qn[2], qn[3]);
  kn4 = make_float4(kn[0], kn[1], kn[2], kn[3]);
  rp = rp < 0 ? 0 : (rp >= S.npos ? S.npos - 1 : rp);
  cs4 = __ldg(reinterpret_cast<const float4*>(S.cos + (size_t)rp * 128) + c.lane);
  sn4 = __ldg(reinterpret_cast<const float4*>(S.sin + (size_t)rp * 128) + c.lane);
}
template <bool BF>
__device__ __forceinline__ void small_kv_preload(Ctx& c, const StackDev& S, int layer, int slot0, int rpos,
                                                 const void* kc, const void* vc, SmallKV<BF>& pre) {
  using Raw = typename SmallKV<BF>::Raw;
  const size_t esz = BF ? 2 : 4;
  const int g = c.warp < S.nKV ? c.warp : 0;
  // all loads go out before the first copy into `pre`: should `pre` ever land in local memory again, a store into it
  // that may alias what a later load's address depends on would serialise the loads (one L2 round trip each)
  const Raw* kp = reinterpret_cast<const Raw*>(reinterpret_cast<const uint8_t*>(kc) + ((size_t)(layer * S.nKV + g) * S.S * 128) * esz) + c.lane;
  const Raw* vp = reinterpret_cast<const Raw*>(reinterpret_cast<const uint8_t*>(vc) + ((size_t)(layer * S.nKV + g) * S.S * 128) * esz) + c.lane;
  constexpr int ROW = (int)(128 * (BF ? 2 : 4) / sizeof(Raw));   // Raw elements per cached row
  Raw k[16], v[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    if (j < slot0) {
      k[j] = __ldcg(kp + j * ROW);
      v[j] = __ldcg(vp + j * ROW);
    } else {
      if constexpr (BF) { k[j] = make_uint2(0, 0); v[j] = make_uint2(0, 0); }
      else { k[j] = make_float4(0, 0, 0, 0); v[j] = make_float4(0, 0, 0, 0); }
    }
  }
  float4 qn, kn, cs, sn;
  if constexpr (BF) small_norm_rope_load<BF>(c, S, layer, rpos, qn, kn, cs, sn);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    pre.k[j] = k[j];
    pre.v[j] = v[j];
  }
  if constexpr (BF) { pre.qn = qn; pre.kn = kn; pre.cs = cs; pre.sn = sn; }
}

//   qkv0: QKV row of token 0, token t lives qkv_tstride floats further; kc / vc: the request's predictor caches;
//   append: this CTA writes the new K/V rows; pre: cached rows already in registers (or nullptr);
//   out(t, i, v): stores element i of token t's attention output (model-dtype rounded)
//   XT: the QKV rows are the tagged exchange `tag`, polled (everything else of round trip 1 is issued first)
template <bool BF, int NT, bool XT = false, class Out>
__device__ void attention_small_all(Ctx& c, const StackDev& S, int layer, int slot0_, int rpos0, const float* __restrict__ qkv0,
                                    size_t qkv_tstride, void* kc, void* vc, bool append, const SmallKV<BF>* pre, Out out,
                                    uint32_t tag = 0) {
  constexpr int NOLD = NT == 2 ? 1 : 16;  // cached keys that can exist
  constexpr int MAXK = NT == 2 ? 2 : 17;
  const int slot0 = NT == 2 ? 0 : slot0_;
  const float scale = 0.08838834764831845f;
  const size_t esz = BF ? 2 : 4;
  const int L4 = 4 * c.lane;
  using Raw = typename std::conditional<BF, uint2, float4>::type;
  auto unpack = [](const Raw& r, float* o) {
    if constexpr (BF) { o[0] = bf_lo(r.x); o[1] = bf_hi(r.x); o[2] = bf_lo(r.y); o[3] = bf_hi(r.y); }
    else { o[0] = r.x; o[1] = r.y; o[2] = r.z; o[3] = r.w; }
  };
  auto zero_raw = [](Raw& r) {
    if constexpr (BF) r = make_uint2(0, 0);
    else r = make_float4(0, 0, 0, 0);
  };
  for (int g = c.warp; g < S.nKV; g += NCW) {
    uint8_t* kb = reinterpret_cast<uint8_t*>(kc) + ((size_t)(layer * S.nKV + g) * S.S * 128) * esz;
    uint8_t* vb = reinterpret_cast<uint8_t*>(vc) + ((size_t)(layer * S.nKV + g) * S.S * 128) * esz;
    // ---- round trip 1: cached K rows + everything about the new token(s)
    Raw kraw[NOLD];
#pragma unroll
    for (int j = 0; j < NOLD; ++j) {
      if (pre && NT == 1 && g == c.warp) kraw[j] = pre->k[j];
      else if (j < slot0) kraw[j] = __ldcg(reinterpret_cast<const Raw*>(kb + (size_t)j * 128 * esz) + c.lane);
      else zero_raw(kraw[j]);
    }
    float4 qn4, kn4, cs4[NT], sn4[NT], kr4[NT], vr4[NT], qr4[2][NT];
    if (BF && pre && NT == 1) {
      qn4 = pre->qn; kn4 = pre->kn; cs4[0] = pre->cs; sn4[0] = pre->sn;
    } else {
#pragma unroll
      for (int t = 0; t < NT; ++t) small_norm_rope_load<BF>(c, S, layer, rpos0 + t, qn4, kn4, cs4[t], sn4[t]);
    }
    auto qkv_at = [&](int t, int which) {   // which: 0, 1 = q of the group's heads, 2 = k, 3 = v
      const float* row = qkv0 + (size_t)t * qkv_tstride;
      return row + (which == 2 ? S.qd + g * 128 : which == 3 ? S.qd + S.kd + g * 128
                                                 : (g * S.rep + (which < S.rep ? which : 0)) * 128) + L4;
    };
    if constexpr (XT) {
      uint4 w[NT][4];
#pragma unroll
      for (int t = 0; t < NT; ++t)
#pragma unroll
        for (int q = 0; q < 4; ++q) w[t][q] = ld_relaxed_v4(qkv_at(t, q));
      auto un = [](const uint4& u) { return make_float4(untag(u.x), untag(u.y), untag(u.z), untag(u.w)); };
#pragma unroll
      for (int t = 0; t < NT; ++t) {
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (!xtag_ok(w[t][q], tag)) w[t][q] = xwait(c.P.xerr, qkv_at(t, q), w[t][q], tag);
        qr4[0][t] = un(w[t][0]); qr4[1][t] = un(w[t][1]); kr4[t] = un(w[t][2]); vr4[t] = un(w[t][3]);
      }
    } else {
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        const float* row = qkv0 + (size_t)t * qkv_tstride;
        kr4[t] = __ldcg(reinterpret_cast<const float4*>(row + S.qd + g * 128) + c.lane);
        vr4[t] = __ldcg(reinterpret_cast<const float4*>(row + S.qd + S.kd + g * 128) + c.lane);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
          qr4[hh][t] = __ldcg(reinterpret_cast<const float4*>(row + (g * S.rep + (hh < S.rep ? hh : 0)) * 128) + c.lane);
      }
    }
    auto norm_rope = [&](float* v, const float4& w4, const float4& c4, const float4& s4) {
      const float w[4] = {w4.x, w4.y, w4.z, w4.w}, cc[4] = {c4.x, c4.y, c4.z, c4.w}, sv[4] = {s4.x, s4.y, s4.z, s4.w};
      float ss = v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3];
#pragma unroll
      for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
      const float r = 1.0f / sqrtf(ss / 128.0f + S.eps);
      float o4[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) v[i] = rnd<BF>(w[i] * rnd<BF>(v[i] * r));
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float other = __shfl_xor_sync(0xffffffffu, v[i], 16);
        const float rot = c.lane < 16 ? -other : other;
        o4[i] = rnd<BF>(rnd<BF>(v[i] * rnd<BF>(cc[i])) + rnd<BF>(rot * rnd<BF>(sv[i])));
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) v[i] = o4[i];
    };
    float knew[NT][4], vnew[NT][4];
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      knew[t][0] = kr4[t].x; knew[t][1] = kr4[t].y; knew[t][2] = kr4[t].z; knew[t][3] = kr4[t].w;
      vnew[t][0] = vr4[t].x; vnew[t][1] = vr4[t].y; vnew[t][2] = vr4[t].z; vnew[t][3] = vr4[t].w;
      norm_rope(knew[t], kn4, cs4[t], sn4[t]);
      if (append) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          stw<BF>(kb + (size_t)(slot0 + t) * 128 * esz, L4 + i, knew[t][i]);
          stw<BF>(vb + (size_t)(slot0 + t) * 128 * esz, L4 + i, vnew[t][i]);
        }
      }
    }
    // ---- scores of every (head, token) of this group; probabilities stay in registers
    float q[2][NT][4];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        q[hh][t][0] = qr4[hh][t].x; q[hh][t][1] = qr4[hh][t].y; q[hh][t][2] = qr4[hh][t].z; q[hh][t][3] = qr4[hh][t].w;
        norm_rope(q[hh][t], qn4, cs4[t], sn4[t]);
      }
    float sc[2][NT][MAXK];
#pragma unroll
    for (int j = 0; j < MAXK; ++j) {
      float kf[4] = {0.f, 0.f, 0.f, 0.f};
      if (j < NOLD && j < slot0) unpack(kraw[j < NOLD ? j : 0], kf);
#pragma unroll
      for (int tn = 0; tn < NT; ++tn)
        if (j == slot0 + tn) {
#pragma unroll
          for (int i = 0; i < 4; ++i) kf[i] = knew[tn][i];
        }
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int t = 0; t < NT; ++t) {
          float d = q[hh][t][0] * kf[0];
          d = fmaf(q[hh][t][1], kf[1], d); d = fmaf(q[hh][t][2], kf[2], d); d = fmaf(q[hh][t][3], kf[3], d);
          sc[hh][t][j] = d;
        }
    }
    float dotk[2] = {0.f, 0.f};   // NT == 1: the full q.k of key `lane` for the two heads (reduce-scatter path)
    if constexpr (NT == 1) {
      float a[34];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int j = 0; j < 17; ++j) a[hh * 17 + j] = sc[hh][0][j];
      rs_step<34, 16>(a, c.lane);
      rs_step<17, 8>(a, c.lane);
      rs_step<9, 4>(a, c.lane);
      rs_step<5, 2>(a, c.lane);
      rs_step<3, 1>(a, c.lane);
      rs34_gather(a, c.lane, dotk);
    } else {
#pragma unroll
      for (int o = 16; o; o >>= 1)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
          for (int t = 0; t < NT; ++t)
#pragma unroll
            for (int j = 0; j < MAXK; ++j) sc[hh][t][j] += __shfl_xor_sync(0xffffffffu, sc[hh][t][j], o);
    }
    // ---- round trip 2: cached V rows (issued before the softmax arithmetic so the latency overlaps it)
    Raw vraw[NOLD];
#pragma unroll
    for (int j = 0; j < NOLD; ++j) {
      if (pre && NT == 1 && g == c.warp) vraw[j] = pre->v[j];
      else if (j < slot0) vraw[j] = __ldcg(reinterpret_cast<const Raw*>(vb + (size_t)j * 128 * esz) + c.lane);
      else zero_raw(vraw[j]);
    }
    // softmax with the keys distributed over lanes: lane j owns key j (its score, its exponential); max and sum are
    // warp reductions and p_j is broadcast with one shuffle per key.
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        const int nk = slot0 + t + 1;
        float mx = -INFINITY, mine = -INFINITY;
        if constexpr (NT == 1) {
          mine = (c.lane < nk) ? rnd<BF>(rnd<BF>(dotk[hh]) * scale) : -INFINITY;
          mx = mine;
#pragma unroll
          for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        } else {
#pragma unroll
          for (int j = 0; j < MAXK; ++j) {
            const float sj = j < nk ? rnd<BF>(rnd<BF>(sc[hh][t][j]) * scale) : -INFINITY;
            mx = fmaxf(mx, sj);
            if (j == c.lane) mine = sj;
          }
        }
        const float e = (c.lane < nk) ? (BF ? __expf(mine - mx) : expf(mine - mx)) : 0.f;
        float sm = e;
#pragma unroll
        for (int o = 16; o; o >>= 1) sm += __shfl_xor_sync(0xffffffffu, sm, o);
        const float pmine = rnd<BF>(BF ? __fdividef(e, sm) : e / sm);
#pragma unroll
        for (int j = 0; j < MAXK; ++j) sc[hh][t][j] = __shfl_sync(0xffffffffu, pmine, j);
      }
    float o4[2][NT][4];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
      for (int t = 0; t < NT; ++t)
#pragma unroll
        for (int i = 0; i < 4; ++i) o4[hh][t][i] = 0.f;
#pragma unroll
    for (int j = 0; j < MAXK; ++j) {
      float vf[4] = {0.f, 0.f, 0.f, 0.f};
      if (j < NOLD && j < slot0) unpack(vraw[j < NOLD ? j : 0], vf);
#pragma unroll
      for (int tn = 0; tn < NT; ++tn)
        if (j == slot0 + tn) {
#pragma unroll
          for (int i = 0; i < 4; ++i) vf[i] = vnew[tn][i];
        }
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int t = 0; t < NT; ++t)
#pragma unroll
          for (int i = 0; i < 4; ++i) o4[hh][t][i] = fmaf(sc[hh][t][j], vf[i], o4[hh][t][i]);
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
      if (hh < S.rep)
#pragma unroll
        for (int t = 0; t < NT; ++t)
#pragma unroll
          for (int i = 0; i < 4; ++i) out(t, (g * S.rep + hh) * 128 + L4 + i, rnd<BF>(o4[hh][t][i]));
  }
  csync();
}

// RMSNorm of a vector (global fp32 or shared fp32) into the staging vector at element offset `off`
constexpr int NORM_E = HMAX / NCT;
// norm weights of one vector into registers (issued in the shadow of a barrier: they are touched once per pass and
// usually miss to HBM, while the activations they scale arrive from L2)
template <bool BF>
__device__ __forceinline__ void norm_wload(Ctx& c, const void* w, size_t woff, int H, float* wv) {
#pragma unroll
  for (int i = 0; i < NORM_E; ++i) {
    const int k = c.tid + i * NCT;
    wv[i] = k < H ? ldw<BF>(w, woff + k) : 0.f;
  }
}
// bf16: a global src is the tagged exchange c.xtag (X or X1), polled
template <bool BF>
__device__ __forceinline__ void norm_stage(Ctx& c, const float* src, bool src_smem, const void* w, size_t woff, int H,
                                           float eps, int off, const float* wpre = nullptr) {
  constexpr int MAXE = NORM_E;
  float v[MAXE], wv[MAXE];
#pragma unroll
  for (int i = 0; i < MAXE; ++i) {
    const int k = c.tid + i * NCT;
    v[i] = 0.f;
    wv[i] = 0.f;
    if (k < H) {
      v[i] = src_smem ? src[k] : (BF ? __uint_as_float(ld_relaxed_u32(src + k)) : __ldcg(src + k));
      wv[i] = wpre ? wpre[i] : ldw<BF>(w, woff + k);
    }
  }
  if (BF && !src_smem) {
#pragma unroll
    for (int i = 0; i < MAXE; ++i) {
      const int k = c.tid + i * NCT;
      uint32_t u = __float_as_uint(v[i]);
      if (k < H && !xtag_ok(u, c.xtag)) u = xwait(c.P.xerr, src + k, u, c.xtag);
      v[i] = untag(u);
    }
  }
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < MAXE; ++i) ss += v[i] * v[i];
  ss = block_sum(c, ss);
  const float r = 1.0f / sqrtf(ss / (float)H + eps);
#pragma unroll
  for (int i = 0; i < MAXE; ++i) {
    const int k = c.tid + i * NCT;
    if (k < H) xs_put<BF>(c, off + k, rnd<BF>(wv[i] * rnd<BF>(v[i] * r)));
  }
  csync();
}

// ------------------------------------------------------------------------------------------------------------
// One pass through a transformer stack for nt tokens held in X (global) or xin (shared, layer 0).
// On return every CTA holds the final-norm hidden of the LAST token in the staging vector [0..H) and X holds the
// residual stream.
// ------------------------------------------------------------------------------------------------------------
// TALKER selects, at compile time, which attention the instantiation contains: the talker's (one q-head per CTA, or
// keys split over several CTAs with TMA-staged K/V) or the predictor's (every CTA computes all heads of the <= 17-key
// cache redundantly).  Two separate real functions: changing one attention cannot perturb the code of the other pass.
template <bool BF, bool TALKER>
__device__ void run_layers(Ctx& c, const StackDev& S, int nt, int slot0, int rpos0, int kv_start,
                                        bool x0_local, bool dbg) {
  constexpr bool is_talker = TALKER;
  const KParams& P = c.P;
  const bool cta0 = blockIdx.x == 0;
  void* kc = P.req.pkc;  // the request's predictor caches (the talker's are paged: P.req.kv / kv_pages)
  void* vc = P.req.pvc;
  int pi = 0;
  dbg = dbg && (P.dbg_on & 1);
  auto nopre = [](int, int) { return 0.f; };
  float wnext[NORM_E];  // norm weights of the NEXT norm, fetched while the preceding barrier is in flight
  for (int l = 0; l < S.L; ++l) {
    probe(c, pi);  // 0: layer start
    // ---- P1: input norm + QKV rows
    for (int t = 0; t < nt; ++t) {
      const float* wp = l > 0 ? wnext : nullptr;
      if (l == 0 && x0_local) norm_stage<BF>(c, SMEM().xin[t], true, S.ln_in, (size_t)l * S.H, S.H, S.eps, t * S.H, wp);
      else norm_stage<BF>(c, P.X + (size_t)t * P.ldX, false, S.ln_in, (size_t)l * S.H, S.H, S.eps, t * S.H, wp);
    }
    probe(c, pi);  // 1: after input norm
    // bf16: QKV, X1 and X are tagged exchanges (B1, B3, B5 are polls, not grid barriers); every CTA advances the tag
    if constexpr (BF) c.xtag = xtag_next(c.xtag);
    const uint32_t xt_qkv = c.xtag;
    gemv_any<BF, false>(c, S.seg_base + 4 * l + 0, nt, S.H, nopre, [&](int row, int t, float v, float, float) {
      xput<BF>(P.QKV + (size_t)t * P.ldQKV + row, rnd<BF>(v), xt_qkv);
    });
    probe(c, pi);  // 2: after QKV gemv
    const bool small_attn = !TALKER;   // geometry checked by fq3_engine_create (cache <= 32 slots, <= 2 q-heads per kv head)
    // a warp preloads its own kv group (warp < nKV); attention_small_all reads further groups (nKV > NCW) itself
    const bool kv_pre = small_attn && nt == 1;
    SmallKV<BF> skv;
    if constexpr (!BF) grid_arrive(c);
    // cached keys/values, norm weights and RoPE rows do not depend on this layer's QKV
    if (kv_pre) small_kv_preload<BF>(c, S, l, slot0, rpos0, kc, vc, skv);
    if constexpr (!BF) grid_wait(c);
    probe(c, pi);  // 3: after B1
    if (dbg && cta0) {
      float* d = P.dbg + (size_t)l * P.dbg_stride_layer;
      for (int t = 0; t < nt; ++t)
        for (int k = c.tid; k < S.qd + 2 * S.kd; k += NCT) {
          const float* q = P.QKV + (size_t)t * P.ldQKV + k;
          d[(size_t)t * (S.qd + 2 * S.kd) + k] = BF ? xload(P.xerr, q, c.xtag) : __ldcg(q);
        }
    }
    if constexpr (!TALKER) {
      // ---- P2+P3 fused: redundant small attention straight into the staging vector (no exchange, no barrier)
      auto to_xs = [&](int t, int i, float v) { xs_put<BF>(c, t * S.qd + i, v); };
      // &skv unconditionally (nt == 1 always preloads): a pointer chosen at run time between skv and nullptr would
      // keep skv in local memory, so that every preloaded row took an STL and an LDL
      if (nt == 1) attention_small_all<BF, 1, BF>(c, S, l, slot0, rpos0, P.QKV, P.ldQKV, kc, vc, cta0, &skv, to_xs, c.xtag);
      else attention_small_all<BF, 2, BF>(c, S, l, slot0, rpos0, P.QKV, P.ldQKV, kc, vc, cta0, nullptr, to_xs, c.xtag);
      probe(c, pi);  // 4
      probe(c, pi);  // 5
    } else {
      // ---- P2: attention of the one talker token.  bf16 talker steps: keys split over attn_split CTAs per q-head, K/V
      //          slices TMA-staged; otherwise one q-head per CTA reading the cache directly
      const bool split = BF && is_talker && nt == 1 && P.attn_split > 0 && slot0 - kv_start >= ATTN_SPLIT_MIN;
      if (split) attention_split<BF>(c, S, l, slot0, rpos0, kv_start);
      else
        for (int h = blockIdx.x; h < S.nH; h += gridDim.x)
          attention_head<BF, BF>(c, S, l, h, P.QKV, P.req.kv, SMEM().kvtab, P.ATT, slot0, rpos0, kv_start, c.xtag);
      if (!split && is_talker && (int)blockIdx.x >= S.nH && slot0 - kv_start > 64) {
        // idle CTAs pull the NEXT layer's keys/values into L2 (evict_last) so the attention CTAs see L2 latency
        const int ln = (l + 1) % S.L;
        const size_t esz = BF ? 2 : 4;
        const int lines_per_row = (int)(128 * esz / 128);
        const int nk = slot0 - kv_start + (ln == 0 ? 1 : 0);
        const long long total = (long long)S.nKV * nk * lines_per_row * 2;
        const int nidle = (int)gridDim.x - S.nH;
        for (long long i = (long long)(blockIdx.x - S.nH) * NCT + c.tid; i < total; i += (long long)nidle * NCT) {
          const int which = (int)(i & 1);
          long long r = i >> 1;
          const int ln_i = (int)(r % lines_per_row);
          r /= lines_per_row;
          const int j = (int)(r % nk);
          const int g = (int)(r / nk);
          const uint8_t* base = kv_row(P.req.kv, S.L, S.nKV, esz, SMEM().kvtab, which, ln, g, kv_start + j) +
                                (size_t)ln_i * 128;
          asm volatile("prefetch.global.L2::evict_last [%0];" ::"l"(base));
        }
      }
      probe(c, pi);  // 4: after attention
      grid_sync(c);
      probe(c, pi);  // 5: after B2
      // ---- P3: o_proj + residual
      // ATT (model dtype, written by other CTAs in this launch: L2-coherent loads, never __ldg) -> staging vector, as
      // raw 16-byte vectors
      {
        const uint4* att = reinterpret_cast<const uint4*>(P.ATT);
        for (int k = c.tid; k < S.qd * (BF ? 2 : 4) / 16; k += NCT) reinterpret_cast<uint4*>(SMEM().xs)[k] = __ldcg(att + k);
      }
      csync();
    }
    if (dbg && cta0) {
      float* d = P.dbg + (size_t)l * P.dbg_stride_layer + (size_t)2 * (S.qd + 2 * S.kd);
      for (int k = c.tid; k < nt * S.qd; k += NCT) d[k] = xs_get<BF>(c, k);
    }
    {
      const bool loc = (l == 0 && x0_local);
      if constexpr (BF) c.xtag = xtag_next(c.xtag);
      const uint32_t xt_x1 = c.xtag;
      gemv_any<BF, false>(
          c, S.seg_base + 4 * l + 1, nt, S.qd,
          [&](int row, int t) { return loc ? SMEM().xin[t][row] : xget<BF>(P.X + (size_t)t * P.ldX + row); },
          [&](int row, int t, float v, float, float res) {
            xput<BF>(P.X1 + (size_t)t * P.ldX + row, rnd<BF>(res + rnd<BF>(v)), xt_x1);
          });
    }
    probe(c, pi);  // 6: after O gemv
    float wpost[NORM_E];
    if constexpr (!BF) grid_arrive(c);
    norm_wload<BF>(c, S.ln_post, (size_t)l * S.H, S.H, wpost);
    if constexpr (!BF) grid_wait(c);
    probe(c, pi);  // 7: after B3
    // ---- P4: post-attention norm + gate/up rows + SiLU*up
    for (int t = 0; t < nt; ++t)
      norm_stage<BF>(c, P.X1 + (size_t)t * P.ldX, false, S.ln_post, (size_t)l * S.H, S.H, S.eps, t * S.H, wpost);
    if (dbg && cta0) {
      float* d = P.dbg + (size_t)l * P.dbg_stride_layer + (size_t)2 * (S.qd + 2 * S.kd) + 2 * S.qd;
      for (int t = 0; t < nt; ++t)
        for (int k = c.tid; k < S.H; k += NCT) d[(size_t)t * S.H + k] = xget<BF>(P.X1 + (size_t)t * P.ldX + k);
    }
    gemv_any<BF, true>(c, S.seg_base + 4 * l + 2, nt, S.H, nopre, [&](int pair, int t, float gv, float uv, float) {
      const float gte = rnd<BF>(gv), up = rnd<BF>(uv);
      const float sl = rnd<BF>(gte / (1.0f + expf(-gte)));
      stw<BF>(P.ACT, (size_t)t * P.ldACT + pair, rnd<BF>(sl * up));   // exact: the value is model-dtype rounded
    });
    probe(c, pi);  // 8: after GU gemv
    grid_sync(c);
    probe(c, pi);  // 9: after B4
    // ---- P5: down rows + residual, reading ACT in place (model dtype, L2-resident; no copy into the staging vector)
    if (dbg && cta0) {
      float* d = P.dbg + (size_t)l * P.dbg_stride_layer + (size_t)2 * (S.qd + 2 * S.kd) + 2 * S.qd + 2 * S.H;
      for (int t = 0; t < nt; ++t)
        for (int k = c.tid; k < S.I; k += NCT) {
          const size_t i = (size_t)t * P.ldACT + k;
          if constexpr (BF) d[(size_t)t * S.I + k] = __bfloat162float(__ldcg(reinterpret_cast<const __nv_bfloat16*>(P.ACT) + i));
          else d[(size_t)t * S.I + k] = __ldcg(reinterpret_cast<const float*>(P.ACT) + i);
        }
    }
    if constexpr (BF) c.xtag = xtag_next(c.xtag);
    const uint32_t xt_x = c.xtag;
    gemv_any<BF, false, true>(
        c, S.seg_base + 4 * l + 3, nt, S.I, [&](int row, int t) { return xget<BF>(P.X1 + (size_t)t * P.ldX + row); },
        [&](int row, int t, float v, float, float res) {
          xput<BF>(P.X + (size_t)t * P.ldX + row, rnd<BF>(res + rnd<BF>(v)), xt_x);
        },
        P.ACT, P.ldACT);
    probe(c, pi);  // 10: after DN gemv
    if constexpr (!BF) grid_arrive(c);
    if (l + 1 < S.L) norm_wload<BF>(c, S.ln_in, (size_t)(l + 1) * S.H, S.H, wnext);
    else norm_wload<BF>(c, S.ln_f, 0, S.H, wnext);
    if constexpr (!BF) grid_wait(c);
    probe(c, pi);  // 11: after B5
    if (dbg && cta0) {
      float* d = P.dbg + (size_t)l * P.dbg_stride_layer + (size_t)2 * (S.qd + 2 * S.kd) + 2 * S.qd + 2 * S.H + 2 * S.I;
      for (int t = 0; t < nt; ++t)
        for (int k = c.tid; k < S.H; k += NCT) {
          const float* x = P.X + (size_t)t * P.ldX + k;
          d[(size_t)t * S.H + k] = BF ? xload(P.xerr, x, c.xtag) : __ldcg(x);
        }
    }
  }
  // final norm of the last token -> staging vector [0..H)
  norm_stage<BF>(c, P.X + (size_t)(nt - 1) * P.ldX, false, S.ln_f, 0, S.H, S.eps, 0, wnext);
}

// head GEMV (rows of a [V,H] matrix) on the staging vector -> LOGITS.  tagged (bf16 predictor): LOGITS is the tagged
// exchange c.xtag, which the sampler polls; otherwise a grid barrier follows.  The talker's head keeps its barrier: the
// next frame's MTP projection writes X with no other barrier in between, and a CTA that owns no head rows may still
// be reading X in the talker's final norm
template <bool BF>
__device__ __forceinline__ void head_logits(Ctx& c, int seg, int H, bool tagged) {
  const KParams& P = c.P;
  if (tagged) c.xtag = xtag_next(c.xtag);
  const uint32_t xt = c.xtag;
  gemv_any<BF, false>(c, seg, 1, H, [](int, int) { return 0.f; }, [&](int row, int, float v, float, float) {
    if (tagged) st_tagged(P.LOGITS + row, rnd<BF>(v), xt);
    else P.LOGITS[row] = rnd<BF>(v);
  });
  if (!tagged) grid_sync(c);
}

// ------------------------------------------------------------------------------------------------------------
// Rules of a frame (generate.py:149-199) that both fq3_decode_kernel and fq3_decode_batch_kernel call.  The stop gate,
// the uniform row, the predictor pass inputs and draws, the talker input and the max_seq_len rule stay written out in
// each kernel: as calls, they raise the spills of one kernel or the other (DESIGN §4).
// ------------------------------------------------------------------------------------------------------------
// the talker's draw (generate.py:46-50): repetition penalty over the seen history; suppress_special: the ids
// [V - 1024, V) other than eos are never drawn; suppress_eos: nor is eos
__device__ __forceinline__ SampleArgs talker_draw(const float* logits, int V, const Sampling& sp, float u,
                                                  bool suppress_special, int eos, bool suppress_eos, float* lp) {
  SampleArgs a;
  a.logits = logits; a.V = V; a.sp = sp; a.u = u;
  a.use_penalty = true; a.sup0 = suppress_special ? (V > 1024 ? V - 1024 : 0) : V;
  a.suppress_eos = suppress_eos; a.eos = eos;
  a.lp = lp;
  return a;
}
// ... of frame `step` of request sp: uniform urow[0], eos held back for the first min_new frames; it writes column 0
// of the frame's log-probability row (the cb0 that follows the frame)
__device__ __forceinline__ SampleArgs frame_talker_draw(const KParams& P, const SlotParams& sp, const float* logits,
                                                        const float* urow, int step, float* lp_row) {
  return talker_draw(logits, P.t.V, sp.sp_t, (sp.sp_t.do_sample && urow) ? __ldg(urow) : 0.f, true, P.eos,
                     step + 1 < sp.min_new, lp_row);
}

// after the talker's draw: its cb0 starts the next frame
__device__ __forceinline__ void frame_advance(int& token, int& step, int& gen_step, int next) {
  token = next;
  ++step;
  ++gen_step;
}

__device__ __forceinline__ void put_state(int* st, int token, int step, int gen_step, int finished, int emitted) {
  st[ST_TOKEN] = token; st[ST_STEP] = step; st[ST_GEN] = gen_step; st[ST_FIN] = finished; st[ST_EMIT] = emitted;
}

// predictor: 15 passes (predictor_graph.py:115-167).  Inputs: s.xin[0] = past_hidden, s.xin[1] = embed(cb0 token).
// Outputs s.codes[1..15].  u15: 15 uniforms.  lp_row: the frame's log-probability row (pass i -> column i + 1) or nullptr.
// A real function that works on a private copy of the caller's Ctx and hands the advanced counters back at the end.
// The caller's Ctx has its address taken and lives in local memory; used directly, every c.lane, c.warp and
// c.tile_ctr of the predictor was an LDL, reloaded after each store the compiler could not prove disjoint from the
// stack (every global store of a GEMV epilogue or a K/V append).  The copy's address is never taken: registers.
// (The caller keeps its own Ctx in memory on purpose: promoted to registers, it adds spills to the talker's path.)
template <bool BF>
__device__ void predictor_frame(Ctx& cio, const float* u15, bool dbg, float* lp_row) {
  Ctx c = cio;
  const KParams& P = c.P;
  const StackDev& S = P.p;
  const int Ht = P.t.H;
  for (int i = 0; i < P.ncb; ++i) {
    const int nt = (i == 0) ? 2 : 1;
    probe_at(c, 1024 + 8 * i + 0);
    // pass 0 projects cat(past_hidden, cb0 embedding), which the table does not cover
    const bool project = i == 0 && P.has_mtp;
    if (project) {
      for (int t = 0; t < nt; ++t)
        for (int k = c.tid; k < Ht; k += NCT) xs_put<BF>(c, t * Ht + k, SMEM().xin[t][k]);
      csync();
      if constexpr (BF) c.xtag = xtag_next(c.xtag);   // bf16: X is a tagged exchange, polled by layer 0's input norm
      const uint32_t xt = c.xtag;
      gemv_any<BF, false>(c, P.seg_mtp, nt, Ht, [&](int row, int) { return P.mtp_b ? ldw<BF>(P.mtp_b, row) : 0.f; },
                          [&](int row, int t, float v, float, float b) {
                            xput<BF>(P.X + (size_t)t * P.ldX + row, rnd<BF>(v + b), xt);
                          });
      if constexpr (!BF) grid_sync(c);
    }
    const int slot0 = (i == 0) ? 0 : i + 1;
    probe_at(c, 1024 + 8 * i + 1);
    run_layers<BF, false>(c, S, nt, slot0, slot0, 0, !project, dbg && i == 0);
    probe_at(c, 1024 + 8 * i + 2);
    head_logits<BF>(c, S.seg_head + i, S.H, BF);
    probe_at(c, 1024 + 8 * i + 3);
    SampleArgs sa;
    sa.logits = P.LOGITS; sa.V = S.V; sa.sp = P.req.sp_p; sa.u = u15 ? __ldg(u15 + i) : 0.f;
    sa.use_penalty = false; sa.sup0 = S.V; sa.suppress_eos = false; sa.eos = -1;
    sa.lp = lp_row ? lp_row + 1 + i : nullptr;
    sa.xtag = BF ? c.xtag : 0u;
    const int tok = sample_block<BF>(c, sa);
    if (c.tid == 0) SMEM().codes[i + 1] = tok;
    if (i + 1 < P.ncb) {
      // the next pass's input row, fetched as soon as the code is known (sample_block is done with xin[0]), all of a
      // thread's loads in flight together.  With the projection: small_to_mtp_projection(codec_embedding[i](tok)),
      // tabulated when the weights were loaded
      const void* tab = P.has_mtp ? P.mtp_tab : P.p_embeds;
      const int n = P.has_mtp ? S.H : Ht;
      float r[NORM_E];
#pragma unroll
      for (int e = 0; e < NORM_E; ++e) {
        const int k = c.tid + e * NCT;
        r[e] = k < n ? ldw<BF>(tab, ((size_t)i * S.V + tok) * n + k) : 0.f;
      }
#pragma unroll
      for (int e = 0; e < NORM_E; ++e) {
        const int k = c.tid + e * NCT;
        if (k < n) SMEM().xin[0][k] = r[e];
      }
    }
    csync();
    probe_at(c, 1024 + 8 * i + 4);
  }
  cio.tile_ctr = c.tile_ctr;
  cio.bar_target = c.bar_target;
  cio.xtag = c.xtag;
}

// ------------------------------------------------------------------------------------------------------------
// The producer warp's whole life, as one real function: its code generation (counters in registers, no spills) must
// not depend on how much register pressure the consumer code around it creates -- a slow producer slows every phase.
// ------------------------------------------------------------------------------------------------------------
template <bool BF>
__device__ __noinline__ void producer_main(const KParams& P) {
  const int lane = (int)(threadIdx.x & 31u);
  if (lane == 0) {
    Producer<BF> pr(P);
    if (P.mode == MODE_TALKER_STEP) pr.stack_layers(P.t, 1, P.position, P.req.n_left_pad);
    else if (P.mode == MODE_PRED_RUN) pr.predictor(1, 1);
    else
      for (int f = 0; f < P.n_frames && !pr.stopped; ++f)
        pr.frame(1, 1, P.req.prefill_len + P.req.state[ST_STEP] + f, P.req.n_left_pad);
    pr.finish();
  }
}

// ------------------------------------------------------------------------------------------------------------
// CTA prologue and drain, shared by fq3_decode_kernel and fq3_decode_batch_kernel
// ------------------------------------------------------------------------------------------------------------
// this CTA's group / segment tables, the cb0 history bitmap (copied from `seen`, zeros when nullptr), the ring
// mbarriers and the hand-shake words; the caller's __syncthreads() publishes them
__device__ __forceinline__ void cta_prologue(const KParams& P, const uint32_t* seen) {
  Smem& s = SMEM();
  const int tid = threadIdx.x, cta = blockIdx.x;
  const uint32_t g0 = __ldg(P.cta_grp_off + cta), g1 = __ldg(P.cta_grp_off + cta + 1);
  for (uint32_t i = tid; i < g1 - g0; i += NTHREADS) s.grp[i] = P.grps[g0 + i];
  for (int i = tid; i < P.nseg; i += NTHREADS) s.seg[i] = __ldg(P.segtab + (size_t)cta * P.nseg + i);
  for (int i = tid; i < VMAX / 32; i += NTHREADS) s.seen[i] = seen ? seen[i] : 0u;
  if (tid == 0) {
    for (int i = 0; i < NS; ++i) {
      mbar_init(&s.full[i], 1);
      mbar_init(&s.empty[i], NCW);
    }
    s.stop_flag = 0;
    s.prod_done = 0;
    s.prod_issued = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
}

// consumers at the end of a launch: stop the producer and wait for every bulk copy it has in flight
__device__ __forceinline__ void drain_producer(Ctx& c) {
  Smem& s = SMEM();
  csync();
  if (c.tid == 0) {
    flag_st(&s.stop_flag, 1);
    __threadfence_block();
    while (!flag_ld(&s.prod_done)) {
    }
    __threadfence_block();
    const uint32_t issued = (uint32_t)flag_ld(&s.prod_issued);
    for (uint32_t t = c.tile_ctr; t < issued; ++t) mbar_wait(&s.full[t % NS], (t / NS) & 1u);
  }
  csync();
}

// ------------------------------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------------------------------
template <bool BF>
__global__ void __launch_bounds__(NTHREADS, 1) fq3_decode_kernel(const __grid_constant__ KParams P) {
  Smem& s = SMEM();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cta = blockIdx.x;

  cta_prologue(P, P.mode == MODE_FUSED ? P.req.seen : nullptr);
  for (int i = tid; i < (P.max_seq_len + KV_PAGE - 1) / KV_PAGE; i += NTHREADS) s.kvtab[i] = P.req.kv_pages[i];
  __syncthreads();

  if (warp == NCW) {
    producer_main<BF>(P);
  } else {
    // ======================================= CONSUMERS ======================================
    Ctx c{P, tid, warp, lane, 0u, 0u};
    const SlotParams& rq = P.req;
    const int Ht = P.t.H;
    if (P.mode == MODE_TALKER_STEP) {
      for (int k = tid; k < Ht; k += NCT) s.xin[0][k] = ldw<BF>(P.in_embeds, k);
      csync();
      run_layers<BF, true>(c, P.t, 1, P.position, P.position + rq.rope_delta, rq.n_left_pad, true, P.dbg_on != 0);
      if (cta == 0)
        for (int k = tid; k < Ht; k += NCT) stw<BF>(P.hidden_out, k, xs_get<BF>(c, k));
    } else if (P.mode == MODE_PRED_RUN) {
      for (int k = tid; k < 2 * Ht; k += NCT) s.xin[k / Ht][k % Ht] = ldw<BF>(P.pred_input, k);
      csync();
      predictor_frame<BF>(c, rq.sp_p.do_sample ? P.pred_uniforms : nullptr, P.dbg_on != 0, nullptr);
      if (cta == 0 && tid < P.ncb) rq.codes_out[tid] = (long long)s.codes[tid + 1];
    } else {
      // ---------------- fused frame loop: generate.py:149-199 / streaming.py:106-173 ----------------
      int token = rq.state[ST_TOKEN], step = rq.state[ST_STEP], gen_step = rq.state[ST_GEN];
      int finished = FQ3_RUNNING, emitted = 0;
      for (int k = tid; k < Ht; k += NCT) s.hid[k] = rq.past_hidden[k];
      csync();
      while (true) {
        if (emitted >= rq.n_frames) break;
        if (step >= rq.max_new) { finished = FQ3_FIN_MAX_NEW; break; }
        if (token == P.eos) { finished = FQ3_FIN_EOS; break; }
        // open text: this frame's talker step reads trailing row gen_step; stop unfinished before touching any state
        if (rq.text_open && gen_step >= rq.trailing_len) break;
        // predictor input: cat(past_hidden, codec_embedding(token))   generate.py:154-155
        for (int k = tid; k < Ht; k += NCT) {
          s.xin[0][k] = s.hid[k];
          s.xin[1][k] = ldw<BF>(P.t_embed, (size_t)token * Ht + k);
        }
        if (tid == 0) {
          s.codes[0] = token;
          s.seen[token >> 5] |= 1u << (token & 31);
        }
        csync();
        const float* urow = rq.uniforms + (size_t)(step + 1) * 16;
        const int pslot = 2048 + 8 * (emitted & 63);
        probe_at(c, pslot + 0);
        // CTA 0 writes the log-probabilities, as it writes the codes
        float* lp_row = (rq.logprob_out && cta == 0) ? rq.logprob_out + (size_t)emitted * 16 : nullptr;
        predictor_frame<BF>(c, rq.sp_p.do_sample ? urow + 1 : nullptr, false, lp_row);
        probe_at(c, pslot + 1);
        if (cta == 0 && tid < 16) rq.codes_out[(size_t)emitted * 16 + tid] = (long long)s.codes[tid];
        emitted++;
        // next talker input: sum of 16 embedding rows + trailing text / tts_pad   generate.py:163-171
        {
          const void* extra = gen_step < rq.trailing_len ? rq.trailing : rq.tts_pad;
          const size_t eoff = gen_step < rq.trailing_len ? (size_t)gen_step * Ht : 0;
          // a thread's NORM_E elements advance through the rows together, so each row is one round of independent
          // loads (not one dependent chain of 16 loads per element); every element still adds its rows in order
          float sm[NORM_E];
#pragma unroll
          for (int e = 0; e < NORM_E; ++e) {
            const int k = tid + e * NCT;
            sm[e] = k < Ht ? ldw<BF>(P.t_embed, (size_t)token * Ht + k) : 0.f;
          }
          for (int i = 0; i < P.ncb; ++i) {
            const size_t row = ((size_t)i * P.p.V + s.codes[i + 1]) * Ht;
#pragma unroll
            for (int e = 0; e < NORM_E; ++e) {
              const int k = tid + e * NCT;
              if (k < Ht) sm[e] += ldw<BF>(P.p_embeds, row + k);
            }
          }
#pragma unroll
          for (int e = 0; e < NORM_E; ++e) {
            const int k = tid + e * NCT;
            if (k < Ht) s.xin[0][k] = rnd<BF>(rnd<BF>(sm[e]) + ldw<BF>(extra, eoff + k));
          }
          csync();
        }
        const int pos = rq.prefill_len + step;
        // generate.py:175-177 (the frame is already emitted)
        if (pos >= P.max_seq_len - 1) { finished = FQ3_FIN_MAX_SEQ; step++; break; }
        probe_at(c, pslot + 2);
        run_layers<BF, true>(c, P.t, 1, pos, pos + rq.rope_delta, rq.n_left_pad, true, false);
        probe_at(c, pslot + 3);
        for (int k = tid; k < Ht; k += NCT) s.hid[k] = xs_get<BF>(c, k);   // past_hidden = post-norm hidden (generate.py:198)
        csync();
        head_logits<BF>(c, P.t.seg_head, Ht, false);
        probe_at(c, pslot + 4);
        const int next = sample_block<BF>(c, frame_talker_draw(P, rq, P.LOGITS, urow, step, lp_row));
        probe_at(c, pslot + 5);
        frame_advance(token, step, gen_step, next);
      }
      if (cta == 0) {
        if (tid == 0) put_state(rq.state, token, step, gen_step, finished, emitted);
        for (int k = tid; k < Ht; k += NCT) rq.past_hidden[k] = s.hid[k];
        for (int i = tid; i < VMAX / 32; i += NCT) rq.seen[i] = s.seen[i];
      }
    }
    drain_producer(c);
  }
  __syncthreads();
}

}  // namespace fq3
