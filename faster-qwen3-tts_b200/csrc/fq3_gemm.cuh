// fq3_gemm.cuh -- channels-last implicit-GEMM kernel shared by the codec stack (K4) and the prefill (K3).
//     Y[t, n] = epilogue( sum_{tap, ci} W[n, tap, ci] * X[t - (taps-1-tap)*dil, ci] )
// 128 x 96 x 32 tiles, 8 warps (2 x 4), bf16 mma.sync m16n8k16 / fp32 accumulation, ldmatrix from XOR-swizzled
// shared memory, 4-stage cp.async pipeline.  Epilogue (all roundings where torch would materialise a bf16 tensor):
//   mode 0: v = rnd(acc + bias); if R: v = rnd(v + R); Yraw <- v; Yact <- SnakeBeta(v)
//           with `scale`: v = rnd(acc + bias) * scale[n] before the residual add (layer scale / ConvNeXt gamma)
//   mode 1: SwiGLU on adjacent column pairs (gate, up): Yraw[t, n/2] = rnd(rnd(silu(rnd(g))) * rnd(u))
//   mode 2: mode 0 with an exact (erf) GELU applied to rnd(acc + bias) first
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

namespace fq3gemm {

// ---- programmatic dependent launch (PDL): the K3 / K4 chains are hundreds of short dependent kernels; with
// programmatic stream serialization kernel N+1 is scheduled as soon as every CTA of kernel N has started, runs its
// prologue (barrier init, tensor-map prefetch) and blocks in griddepcontrol.wait
// until kernel N has completed and flushed its memory -- launch latency and prologue leave the critical path, memory
// semantics are those of ordinary stream order.  Every kernel launched through launch_pdl() calls pdl_wait() before
// its first access to memory another kernel may have written.  FQ3_NO_PDL=1 launches them plainly (A/B).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
static inline bool pdl_enabled() {
  static const bool on = [] {
    const char* v = getenv("FQ3_NO_PDL");
    return !(v && atoi(v) != 0);
  }();
  return on;
}
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                     Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#define FQ3_LAUNCH(kernel, grid, block, smem, stream, ...) \
  fq3gemm::launch_pdl(kernel, dim3(grid), dim3(block), (size_t)(smem), stream, __VA_ARGS__)

constexpr int BM = 128, BN = 96, BK = 32, STAGES = 4, CTHREADS = 256;
constexpr int A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2;
constexpr int CONV_SMEM = STAGES * (A_BYTES + B_BYTES);

struct ConvArgs {
  const __nv_bfloat16* X;   // [T][Cin]
  const __nv_bfloat16* W;   // [N][taps][Cin]
  const float* bias;        // [bias_mod] or null
  const __nv_bfloat16* R;   // residual [T][N] or null
  __nv_bfloat16* Yraw;      // [T][N] or null
  __nv_bfloat16* Yact;      // [T][N] or null
  const float* ea;          // exp(alpha) [act_mod]
  const float* ib;          // 1 / (exp(beta) + 1e-9) [act_mod]
  int T, Cin, N, taps, dil, bias_mod, act_mod;
  int mode;                 // 0 general, 1 SwiGLU pair epilogue (Yraw is [T][N/2]), 2 general with GELU
  const float* scale;       // per-column factor [scale_mod] applied to rnd(acc + bias) before the residual, or null
  int scale_mod;
  // stateful streaming (history rows in front of the new ones): X is [batch][x_rows][Cin] and output row m reads input
  // rows x_row0 + m - shift; rows outside [0, x_rows) read as zero.  x_rows == 0 means x_rows = T, x_row0 = 0.
  int x_row0, x_rows;
  int batch;                // independent sequences: X is [batch][T][Cin], R / Yraw / Yact are [batch][T][N]; every
                            // sequence has its own causal left padding (0 or 1 = a single sequence)
};

__device__ __forceinline__ uint32_t s_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;  // src-size 0 => zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s_u32(dst)), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void ldsm4(uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "r"(s_u32(p)));
}
__device__ __forceinline__ void ldsm2(uint32_t& a, uint32_t& b, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];" : "=r"(a), "=r"(b) : "r"(s_u32(p)));
}
__device__ __forceinline__ void mma16816(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
// swizzled byte offset of (row, 16-byte chunk) inside a [rows][32 bf16] tile
__device__ __forceinline__ int swz(int row, int chunk) { return row * 64 + ((chunk ^ ((row >> 1) & 3)) << 4); }

static __global__ void __launch_bounds__(CTHREADS, 2) conv_gemm_kernel(  // static: included by two TUs
    const __grid_constant__ ConvArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  pdl_launch();
  pdl_wait();
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_BYTES;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wm = warp >> 2, wn = warp & 3;  // 2 x 4 warps; warp tile 64 x 24
  const int tiles_m = (a.T + BM - 1) / BM;
  const int bidx = blockIdx.x / tiles_m;     // sequence of the batch
  const int m0 = (blockIdx.x - bidx * tiles_m) * BM, n0 = blockIdx.y * BN;
  const int kc = a.Cin / BK;                 // k-steps per tap
  const int nks = a.taps * kc;
  const int xrows = a.x_rows > 0 ? a.x_rows : a.T;
  const __nv_bfloat16* Xb = a.X + (size_t)bidx * xrows * a.Cin;
  const size_t ybase = (size_t)bidx * a.T * a.N;

  auto load_stage = [&](int ks, int stage) {
    const int tap = ks / kc, c0 = (ks - tap * kc) * BK;
    const int shift = (a.taps - 1 - tap) * a.dil;
    uint8_t* A = sA + stage * A_BYTES;
    uint8_t* B = sB + stage * B_BYTES;
#pragma unroll
    for (int i = 0; i < 2; ++i) {  // 128 rows x 4 chunks
      const int q = tid + i * CTHREADS;
      const int row = q >> 2, ch = q & 3;
      const int t = m0 + row - shift + a.x_row0;
      const bool ok = t >= 0 && t < xrows && (m0 + row) < a.T;
      const __nv_bfloat16* src = Xb + ((size_t)(ok ? t : 0) * a.Cin + c0 + ch * 8);
      cp_async16(A + swz(row, ch), src, ok);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {  // 96 rows x 4 chunks = 384
      const int q = tid + i * CTHREADS;
      if (q < BN * 4) {
        const int row = q >> 2, ch = q & 3;
        const int n = n0 + row;
        const bool ok = n < a.N;
        const __nv_bfloat16* src = a.W + (((size_t)(ok ? n : 0) * a.taps + tap) * a.Cin + c0 + ch * 8);
        cp_async16(B + swz(row, ch), src, ok);
      }
    }
  };

  float acc[4][3][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[i][j][r] = 0.f;

#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < nks) load_stage(s, s);
    cp_commit();
  }
  for (int ks = 0; ks < nks; ++ks) {
    cp_wait<STAGES - 2>();
    __syncthreads();
    {
      const int nx = ks + STAGES - 1;
      if (nx < nks) load_stage(nx, nx % STAGES);
      cp_commit();
    }
    const uint8_t* A = sA + (ks % STAGES) * A_BYTES;
    const uint8_t* B = sB + (ks % STAGES) * B_BYTES;
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {  // two k16 steps per BK
      uint32_t af[4][4];
#pragma unroll
      for (int mi = 0; mi < 4; ++mi) {
        const int row = wm * 64 + mi * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
        const int ch = kk * 2 + (lane >> 4);
        ldsm4(af[mi][0], af[mi][1], af[mi][2], af[mi][3], A + swz(row, ch));
      }
      uint32_t bf[3][2];
      {
        // n-tiles 0,1 via x4: matrices (n 0-7,k lo) (n 0-7,k hi) (n 8-15,k lo) (n 8-15,k hi)
        const int row = wn * 24 + (lane & 7) + ((lane >> 4) & 1) * 8;
        const int ch = kk * 2 + ((lane >> 3) & 1);
        ldsm4(bf[0][0], bf[0][1], bf[1][0], bf[1][1], B + swz(row, ch));
        const int row2 = wn * 24 + 16 + (lane & 7);
        const int ch2 = kk * 2 + ((lane >> 3) & 1);
        ldsm2(bf[2][0], bf[2][1], B + swz(row2, ch2));
      }
#pragma unroll
      for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int ni = 0; ni < 3; ++ni) mma16816(acc[mi][ni], af[mi], bf[ni][0], bf[ni][1]);
    }
  }
  cp_wait<0>();

  // ---- epilogue: bias, residual, raw / SnakeBeta-activated outputs (bf16x2 stores)
  const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
  for (int mi = 0; mi < 4; ++mi) {
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int m = m0 + wm * 64 + mi * 16 + g + half * 8;
      if (m >= a.T) continue;
#pragma unroll
      for (int ni = 0; ni < 3; ++ni) {
        const int n = n0 + wn * 24 + ni * 8 + t4 * 2;
        if (n >= a.N) continue;
        float v0 = acc[mi][ni][half * 2 + 0], v1 = acc[mi][ni][half * 2 + 1];
        if (a.mode == 1) {
          const float gte = __bfloat162float(__float2bfloat16_rn(v0)), up = __bfloat162float(__float2bfloat16_rn(v1));
          const float sl = __bfloat162float(__float2bfloat16_rn(gte / (1.0f + expf(-gte))));
          a.Yraw[(ybase >> 1) + (size_t)m * (a.N >> 1) + (n >> 1)] = __float2bfloat16_rn(sl * up);
          continue;
        }
        if (a.bias) {
          v0 += a.bias[n % a.bias_mod];
          v1 += a.bias[(n + 1) % a.bias_mod];
        }
        if (a.mode == 2) {
          v0 = gelu_erf(__bfloat162float(__float2bfloat16_rn(v0)));
          v1 = gelu_erf(__bfloat162float(__float2bfloat16_rn(v1)));
        }
        if (a.scale) {
          v0 = __bfloat162float(__float2bfloat16_rn(v0)) * a.scale[n % a.scale_mod];
          v1 = __bfloat162float(__float2bfloat16_rn(v1)) * a.scale[(n + 1) % a.scale_mod];
        }
        const size_t off = ybase + (size_t)m * a.N + n;
        if (a.R) {  // torch: conv/linear output is a bf16 tensor, THEN the residual add (second rounding)
          const __nv_bfloat162 r = *reinterpret_cast<const __nv_bfloat162*>(a.R + off);
          v0 = __bfloat162float(__float2bfloat16_rn(v0)) + __bfloat162float(r.x);
          v1 = __bfloat162float(__float2bfloat16_rn(v1)) + __bfloat162float(r.y);
        }
        // the tensor the next layer sees is bf16: round first, activate the rounded value
        const __nv_bfloat162 raw = __floats2bfloat162_rn(v0, v1);
        if (a.Yraw) *reinterpret_cast<__nv_bfloat162*>(a.Yraw + off) = raw;
        if (a.Yact) {
          const float x0 = __bfloat162float(raw.x), x1 = __bfloat162float(raw.y);
          const int c0 = n % a.act_mod, c1 = (n + 1) % a.act_mod;
          const float s0 = __sinf(x0 * a.ea[c0]), s1 = __sinf(x1 * a.ea[c1]);
          *reinterpret_cast<__nv_bfloat162*>(a.Yact + off) =
              __floats2bfloat162_rn(x0 + a.ib[c0] * s0 * s0, x1 + a.ib[c1] * s1 * s1);
        }
      }
    }
  }
}


}  // namespace fq3gemm
