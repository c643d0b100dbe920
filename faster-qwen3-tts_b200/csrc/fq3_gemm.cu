// fq3_gemm.cu -- fq3gemm::gemm(), the implicit-GEMM causal conv / linear layer of K3 and K4 (arguments and epilogue
// semantics: fq3_gemm.cuh), on Hopper tensor cores (sm_90a):
//   * operands staged by TMA (cp.async.bulk.tensor.2d/3d, SASS UTMALDG) into 128B/64B-swizzled shared-memory tiles;
//     the causal left padding and the M/N tails are TMA out-of-bounds zero fill (negative row coordinates),
//   * warp-specialised: warps 0-3 form one consumer warpgroup that issues wgmma.mma_async m64n96k16 (SASS HGMMA,
//     both operands read from shared memory through matrix descriptors, 128 x 96 fp32 accumulator in registers) and
//     then runs the epilogue; warp 4 is the TMA producer,
//   * one 128 x 96 output tile per CTA; full/empty mbarrier ring of 3 (BK=64) / 4 (BK=32) stages sized so 2-3 CTAs
//     co-reside per SM, or 7 / 12 stages for grids that do not fill the machine,
//   * epilogue: the accumulator is staged through shared memory so that each consumer thread owns one output row
//     (bias / residual / SnakeBeta / SwiGLU -> 16-byte bf16 stores).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <mutex>
#include <unordered_map>

#include "fq3_gemm.cuh"

namespace fq3tc {

constexpr int TBM = 128, TBN = 96, TTHREADS = 160;   // warps 0-3: consumer warpgroup, warp 4: TMA producer
constexpr int SC_LD = TBN + 1;                        // fp32 staging row stride (odd: row-per-thread reads hit 32 banks)
constexpr int SC_BYTES = TBM * SC_LD * 4;

// KIND 0: small ring, so 2-3 CTAs co-reside per SM and overlap each other's prologue / epilogue;
// KIND 1: deep ring, for grids that do not fill the machine (latency-bound main loop).
template <int BK, int KIND>
struct Cfg {
  static constexpr int A_BYTES = TBM * BK * 2;
  static constexpr int B_BYTES = TBN * BK * 2;
  static constexpr int STAGE = A_BYTES + B_BYTES;
  static constexpr int STAGES = KIND == 1 ? (BK == 64 ? 7 : 12) : (BK == 64 ? 3 : 4);
  static constexpr int RING = STAGES * STAGE;
  static constexpr int EP_OFF = RING + 256 /*barriers*/;
  static constexpr int SMEM = 1024 /*align slack*/ + EP_OFF + 4 * TBN * 4 /*epilogue params*/;
  static constexpr uint32_t SBO = (8 * BK * 2) >> 4;          // 8-row group stride, 16-byte units
  static constexpr uint64_t LAYOUT = BK == 64 ? 1ull : 2ull;  // wgmma descriptor: SWIZZLE_128B : SWIZZLE_64B
  static constexpr uint32_t A_HALF = (64 * BK * 2) >> 4;      // rows 64..127 of the A tile, 16-byte units
  static_assert(RING >= SC_BYTES, "accumulator staging must fit in the ring");
  static_assert(2 * STAGES * 8 <= 256, "barriers exceed their slot");
  static_assert(SMEM <= 232448, "exceeds the 227 KB per-CTA shared-memory limit");
};

__device__ __forceinline__ uint32_t su32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mb_init(uint64_t* b, uint32_t n) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(su32(b)), "r"(n) : "memory");
}
__device__ __forceinline__ void mb_expect(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(su32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mb_arrive(uint64_t* b) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(su32(b)) : "memory");
}
// bounded wait: a descriptor / protocol bug traps instead of hanging the GPU
__device__ __forceinline__ void mb_wait(uint64_t* b, uint32_t parity) {
  const long long t0 = clock64();
  while (true) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(su32(b)), "r"(parity) : "memory");
    if (ok) return;
    if (clock64() - t0 > 4000000000ll) __trap();
  }
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* tm, int c0, int c1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(su32(dst)), "l"(tm), "r"(su32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* tm, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
               ::"r"(su32(dst)), "l"(tm), "r"(su32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// wgmma matrix descriptor of a K-major swizzled tile (tiles are 1024-byte aligned: base offset 0)
__device__ __forceinline__ uint64_t smem_desc(const void* p, uint32_t sbo, uint64_t layout) {
  uint64_t d = 0;
  d |= (uint64_t)((su32(p) >> 4) & 0x3fff);   // start address
  d |= (uint64_t)1 << 16;                     // leading byte offset (unused for swizzled K-major) = 1
  d |= (uint64_t)(sbo & 0x3fff) << 32;        // stride byte offset
  d |= layout << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// d[64 x 96] (+)= A[64 x 16] * B[96 x 16]^T, bf16 operands K-major in shared memory, fp32 accumulator
__device__ __forceinline__ void wgmma_m64n96(float (&d)[48], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,"
      "%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47}, %48, %49, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "l"(da), "l"(db), "r"(acc)
      : "memory");
}

// epilogue of one accumulator row (r: 96 fp32 columns of output row m of sequence bidx, columns n0..n0+95);
// ep: [4][TBN] staged bias / exp(alpha) / 1/(exp(beta)+eps) / scale of these columns
__device__ __forceinline__ void tc_epilogue_row(const fq3gemm::ConvArgs& a, const float* ep, uint32_t (&r)[3][32], int m,
                                                int bidx, int n0) {
if (m < a.T) {
  if (a.mode == 1) {
    __nv_bfloat16* dst = a.Yraw + ((size_t)bidx * a.T + m) * (a.N >> 1) + (n0 >> 1);
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      __align__(16) __nv_bfloat16 o[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float gte = __bfloat162float(__float2bfloat16_rn(__uint_as_float(r[j][2 * i])));
        const float up = __bfloat162float(__float2bfloat16_rn(__uint_as_float(r[j][2 * i + 1])));
        const float sl = __bfloat162float(__float2bfloat16_rn(gte / (1.0f + expf(-gte))));
        o[i] = __float2bfloat16_rn(sl * up);
      }
      if (n0 + j * 32 < a.N) {
        *reinterpret_cast<uint4*>(dst + j * 16) = *reinterpret_cast<const uint4*>(o);
        *reinterpret_cast<uint4*>(dst + j * 16 + 8) = *reinterpret_cast<const uint4*>(o + 8);
      }
    }
  } else {
    const size_t off = ((size_t)bidx * a.T + m) * a.N + n0;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
#pragma unroll
      for (int h = 0; h < 4; ++h) {  // 8 columns at a time (16-byte vectors)
        const int n = n0 + j * 32 + h * 8;
        if (n >= a.N) continue;
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = __uint_as_float(r[j][h * 8 + i]);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] += ep[j * 32 + h * 8 + i];
        if (a.mode == 2) {
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] = fq3gemm::gelu_erf(__bfloat162float(__float2bfloat16_rn(v[i])));
        }
        if (a.scale) {
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] = __bfloat162float(__float2bfloat16_rn(v[i])) * ep[3 * TBN + j * 32 + h * 8 + i];
        }
        if (a.R) {
          const uint4 rr = *reinterpret_cast<const uint4*>(a.R + off + j * 32 + h * 8);
          const __nv_bfloat16* rb = reinterpret_cast<const __nv_bfloat16*>(&rr);
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] = __bfloat162float(__float2bfloat16_rn(v[i])) + __bfloat162float(rb[i]);
        }
        __align__(16) __nv_bfloat16 raw[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) raw[i] = __float2bfloat16_rn(v[i]);
        if (a.Yraw) *reinterpret_cast<uint4*>(a.Yraw + off + j * 32 + h * 8) = *reinterpret_cast<const uint4*>(raw);
        if (a.Yact) {
          __align__(16) __nv_bfloat16 act[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float x = __bfloat162float(raw[i]);
            const int cidx = j * 32 + h * 8 + i;
            const float sn = __sinf(x * ep[TBN + cidx]);
            act[i] = __float2bfloat16_rn(x + ep[2 * TBN + cidx] * sn * sn);
          }
          *reinterpret_cast<uint4*>(a.Yact + off + j * 32 + h * 8) = *reinterpret_cast<const uint4*>(act);
        }
      }
    }
  }
}
}

// One CTA per tile.  Tiles are numbered M fastest (tile = nt * tiles_mb + bidx * tiles_m + m-tile), so the CTAs running
// concurrently share one weight tile (L2 / TMA locality).
template <int BK, int KIND>
static __global__ void __launch_bounds__(TTHREADS, KIND == 0 ? 2 : 1)
    conv_gemm_tc_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW,
                        const __grid_constant__ fq3gemm::ConvArgs a, const int tiles_m, const int tiles_mb) {
  using C = Cfg<BK, KIND>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* tiles = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(tiles + C::RING);
  uint64_t* empty = full + C::STAGES;
  float* ep = reinterpret_cast<float*>(tiles + C::EP_OFF);  // [4][TBN]: bias, exp(alpha), 1/(exp(beta)+eps), scale
  float* sc = reinterpret_cast<float*>(tiles);              // [TBM][SC_LD] fp32 accumulator tile, in the drained ring
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kc = a.Cin / BK, nks = a.taps * kc;
  const int nt = blockIdx.x / tiles_mb, mb = blockIdx.x - nt * tiles_mb;
  const int bidx = mb / tiles_m, m0 = (mb - bidx * tiles_m) * TBM, n0 = nt * TBN;

  if (threadIdx.x == 0) {
    for (int i = 0; i < C::STAGES; ++i) { mb_init(&full[i], 1); mb_init(&empty[i], 128); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmX) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmW) : "memory");
  }
  __syncthreads();
  fq3gemm::pdl_launch();   // the next kernel of the chain may start its own prologue ...
  fq3gemm::pdl_wait();     // ... and this one touches activations only after its predecessor has completed

  if (warp == 4) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      for (int ks = 0; ks < nks; ++ks) {
        const int s = ks % C::STAGES;
        mb_wait(&empty[s], ((ks / C::STAGES) & 1u) ^ 1u);
        const int tap = ks / kc, c0 = (ks - tap * kc) * BK;
        const int shift = (a.taps - 1 - tap) * a.dil;
        uint8_t* A = tiles + s * C::STAGE;
        mb_expect(&full[s], C::STAGE);
        tma_load_3d(A, &tmX, c0, m0 - shift + a.x_row0, bidx, &full[s]);   // rows < 0 or >= T of this sequence are zero-filled by TMA
        tma_load_2d(A + C::A_BYTES, &tmW, tap * a.Cin + c0, n0, &full[s]);
      }
    }
    return;
  }

  // ===================== consumer warpgroup: wgmma main loop + epilogue =====================
  const int t = threadIdx.x;   // 0..127
  // per-column parameters of this tile go to shared memory while the first stages are in flight
  for (int i = t; i < TBN; i += 128) {
    const int n = n0 + i;
    const bool ok = n < a.N && a.mode != 1;
    ep[i] = (ok && a.bias) ? a.bias[n % a.bias_mod] : 0.f;
    ep[TBN + i] = (ok && a.Yact) ? a.ea[n % a.act_mod] : 0.f;
    ep[2 * TBN + i] = (ok && a.Yact) ? a.ib[n % a.act_mod] : 0.f;
    ep[3 * TBN + i] = (ok && a.scale) ? a.scale[n % a.scale_mod] : 1.f;
  }
  float acc[2][48];   // rows 0-63 / 64-127 of the tile
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < 48; ++i) acc[h][i] = 0.f;
  for (int ks = 0; ks < nks; ++ks) {
    const int s = ks % C::STAGES;
    mb_wait(&full[s], (ks / C::STAGES) & 1u);
    const uint8_t* A = tiles + s * C::STAGE;
    const uint64_t da = smem_desc(A, C::SBO, C::LAYOUT), db = smem_desc(A + C::A_BYTES, C::SBO, C::LAYOUT);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {  // advance 16 elements = 32 bytes = 2 x 16-byte units along K
      wgmma_m64n96(acc[0], da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (ks | k) ? 1u : 0u);
      wgmma_m64n96(acc[1], da + (uint64_t)(C::A_HALF + 2 * k), db + (uint64_t)(2 * k), (ks | k) ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<1>();                                            // the previous stage's MMAs have read their operands
    if (ks > 0) mb_arrive(&empty[(ks - 1) % C::STAGES]);
  }
  wgmma_wait<0>();
  asm volatile("bar.sync 1, 128;" ::: "memory");   // all MMAs of the warpgroup are done before the staging buffer is written
  {
    // accumulator fragment: register 4j + 2h + c holds row 16 * warp + lane / 4 + 8h, column 8j + 2 (lane % 4) + c
    const int r0 = warp * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int hm = 0; hm < 2; ++hm)
#pragma unroll
      for (int j = 0; j < 12; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int c = 0; c < 2; ++c) sc[(hm * 64 + r0 + 8 * h) * SC_LD + 8 * j + c0 + c] = acc[hm][4 * j + 2 * h + c];
  }
  asm volatile("bar.sync 1, 128;" ::: "memory");
  uint32_t r[3][32];
#pragma unroll
  for (int j = 0; j < 3; ++j)
#pragma unroll
    for (int i = 0; i < 32; ++i) r[j][i] = __float_as_uint(sc[t * SC_LD + j * 32 + i]);
  tc_epilogue_row(a, ep, r, m0 + t, bidx, n0);
}

// ---- host side: tensor maps through the driver entry point (no -lcuda needed) ------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}
// 2-D bf16 row-major [rows][cols] with box [box_rows][box_cols]; swizzle = span of box_cols (64 -> 128B, 32 -> 64B)
static bool make_map(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows, uint32_t box_cols) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return false;
  const cuuint64_t dims[2] = {cols, rows};
  const cuuint64_t strides[1] = {cols * 2};
  const cuuint32_t box[2] = {box_cols, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUtensorMapSwizzle sw = box_cols == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  return fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// 3-D bf16 [batch][rows][cols] with box [1][box_rows][box_cols]: out-of-range rows of ONE sequence read as zero
static bool make_map3(CUtensorMap* tm, const void* base, uint64_t batch, uint64_t rows, uint64_t cols, uint32_t box_rows,
                      uint32_t box_cols) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return false;
  const cuuint64_t dims[3] = {cols, rows, batch};
  const cuuint64_t strides[2] = {cols * 2, rows * cols * 2};
  const cuuint32_t box[3] = {box_cols, box_rows, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  const CUtensorMapSwizzle sw = box_cols == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  return fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Tensor maps are pure functions of (base, shape, box): encode each distinct one ONCE and reuse it on every later
// launch (weights and the engine's activation buffers keep their addresses), so a launch costs no driver call.
struct MapKey {
  const void* base;
  uint64_t batch, rows, cols;
  uint32_t box_rows, box_cols;
  bool operator==(const MapKey& o) const {
    return base == o.base && batch == o.batch && rows == o.rows && cols == o.cols && box_rows == o.box_rows && box_cols == o.box_cols;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    uint64_t h = (uint64_t)(uintptr_t)k.base * 0x9e3779b97f4a7c15ull;
    h ^= (k.rows + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2));
    h ^= (k.cols * 1315423911ull + (h << 6) + (h >> 2));
    h ^= ((k.batch << 40) ^ ((uint64_t)k.box_rows << 20) ^ k.box_cols) + (h << 6) + (h >> 2);
    return (size_t)h;
  }
};
static bool cached_map(CUtensorMap* tm, const void* base, uint64_t batch /*0: 2-D*/, uint64_t rows, uint64_t cols,
                       uint32_t box_rows, uint32_t box_cols) {
  static std::mutex mu;
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  const MapKey key{base, batch, rows, cols, box_rows, box_cols};
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(key);
  if (it != cache.end()) {
    *tm = it->second;
    return true;
  }
  const bool ok = batch ? make_map3(tm, base, batch, rows, cols, box_rows, box_cols) : make_map(tm, base, rows, cols, box_rows, box_cols);
  if (!ok) return false;
  if (cache.size() > 16384) cache.clear();
  cache.emplace(key, *tm);
  return true;
}

template <int BK, int KIND>
static bool set_smem_attr() {
  return cudaFuncSetAttribute(conv_gemm_tc_kernel<BK, KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<BK, KIND>::SMEM) == cudaSuccess;
}
template <int BK, int KIND>
static void launch_kind(const CUtensorMap& tmX, const CUtensorMap& tmW, const fq3gemm::ConvArgs& a, int tiles_m,
                        int tiles_mb, int ntiles, cudaStream_t stream) {
  FQ3_LAUNCH((conv_gemm_tc_kernel<BK, KIND>), ntiles, TTHREADS, (Cfg<BK, KIND>::SMEM), stream, tmX, tmW, a, tiles_m, tiles_mb);
}

}  // namespace fq3tc

const char* fq3gemm::gemm(const ConvArgs& a, cudaStream_t stream) {
  using namespace fq3tc;
  static bool attr_done = false;
  static int num_sms = 132;
  if (!attr_done) {
    if (!set_smem_attr<64, 0>() || !set_smem_attr<32, 0>() || !set_smem_attr<64, 1>() || !set_smem_attr<32, 1>())
      return cudaGetErrorString(cudaGetLastError());
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
    attr_done = true;
  }
  const int BK = (a.Cin % 64 == 0) ? 64 : ((a.Cin % 32 == 0) ? 32 : 0);
  if (!BK || (a.mode == 1 ? (a.N % 32 != 0) : (a.N % 8 != 0))) return "shape unsupported (Cin % 32, N % 8, SwiGLU N % 32)";
  if (((uintptr_t)a.X | (uintptr_t)a.W | (uintptr_t)a.R | (uintptr_t)a.Yraw | (uintptr_t)a.Yact) & 15)
    return "operand not 16-byte aligned";
  const int nb = a.batch > 1 ? a.batch : 1;
  const long long tiles_m = (a.T + TBM - 1) / TBM, tiles_mb = tiles_m * nb;
  const long long ntiles = tiles_mb * ((a.N + TBN - 1) / TBN);
  if (ntiles >= (1ll << 30)) return "too many output tiles";
  CUtensorMap tmX, tmW;
  if (!cached_map(&tmX, a.X, (uint64_t)nb, (uint64_t)(a.x_rows > 0 ? a.x_rows : a.T), (uint64_t)a.Cin, TBM, BK) ||
      !cached_map(&tmW, a.W, 0, (uint64_t)a.N, (uint64_t)a.taps * a.Cin, TBN, BK))
    return "TMA tensor-map encoding failed";
  const int tm = (int)tiles_m, tmb = (int)tiles_mb, nt = (int)ntiles;
  if (ntiles <= (long long)num_sms * 3 / 2) {
    if (BK == 64) launch_kind<64, 1>(tmX, tmW, a, tm, tmb, nt, stream);
    else launch_kind<32, 1>(tmX, tmW, a, tm, tmb, nt, stream);
  } else {
    if (BK == 64) launch_kind<64, 0>(tmX, tmW, a, tm, tmb, nt, stream);
    else launch_kind<32, 0>(tmX, tmW, a, tm, tmb, nt, stream);
  }
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}
