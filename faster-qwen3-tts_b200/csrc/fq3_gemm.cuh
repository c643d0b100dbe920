// fq3_gemm.cuh -- the dense-layer entry point shared by the codec (K4) and the prefill (K3), and the device helpers
// both use.  fq3gemm::gemm() is a channels-last implicit GEMM (a causal conv1d; taps = 1 is a linear layer):
//     Y[t, n] = epilogue( sum_{tap, ci} W[n, tap, ci] * X[t - (taps-1-tap)*dil, ci] )
// It runs the wgmma / TMA kernel of fq3_gemm.cu.  Epilogue (all roundings where torch would materialise a bf16 tensor):
//   mode 0: v = rnd(acc + bias); if R: v = rnd(v + R); Yraw <- v; Yact <- SnakeBeta(v)
//           with `scale`: v = rnd(acc + bias) * scale[n] before the residual add (layer scale / ConvNeXt gamma)
//   mode 1: SwiGLU on adjacent column pairs (gate, up): Yraw[t, n/2] = rnd(rnd(silu(rnd(g))) * rnd(u))
//   mode 2: mode 0 with an exact (erf) GELU applied to rnd(acc + bias) first
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

namespace fq3gemm {

// ---- programmatic dependent launch (PDL): the K3 / K4 chains are hundreds of short dependent kernels; with
// programmatic stream serialization kernel N+1 is scheduled as soon as every CTA of kernel N has started, runs its
// prologue (barrier init, tensor-map prefetch) and blocks in griddepcontrol.wait
// until kernel N has completed and flushed its memory -- launch latency and prologue leave the critical path, memory
// semantics are those of ordinary stream order.  Every kernel launched through launch_pdl() calls pdl_wait() before
// its first access to memory another kernel may have written.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
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
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#define FQ3_LAUNCH(kernel, grid, block, smem, stream, ...) \
  fq3gemm::launch_pdl(kernel, dim3(grid), dim3(block), (size_t)(smem), stream, __VA_ARGS__)

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

// Launches the GEMM on `stream`.  Requires Cin % 32 == 0, N % 8 == 0 (N % 32 == 0 in mode 1) and 16-byte aligned
// X / W / R / Yraw / Yact; callers refuse other shapes when their weights load.  Returns nullptr on success, else a
// description of the failure.
const char* gemm(const ConvArgs& a, cudaStream_t stream);

__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;  // src-size 0 => zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src),
               "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

}  // namespace fq3gemm
