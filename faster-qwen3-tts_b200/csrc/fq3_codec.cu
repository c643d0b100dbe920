// fq3_codec.cu -- K4: the waveform decoder stack of the codec (conv_in -> 4 x [SnakeBeta, causal ConvTranspose,
// 3 residual units] -> SnakeBeta -> conv_out -> clamp) as hand-written sm_90a kernels behind the C ABI.
// Replaces the cuDNN/cuBLAS launches issued by the reference's `speech_tokenizer.decode` call sites
// (faster_qwen3_tts/model.py:924,1093,1122) for the FLOP-dominant part of the decoder (94% of its FLOPs).
//
// One kernel does every dense layer: a causal conv1d as an implicit GEMM over channels-last bf16 activations
//     Y[t, n] = bias[n] + sum_{tap, ci} W[n, tap, ci] * X[t - (taps-1-tap)*dil, ci]        (X[<0] = 0)
//   * M = time, N = output channels, K = taps x Cin; fq3gemm::gemm (fq3_gemm.cu): 128 x 96 tiles, wgmma with fp32
//     accumulation, TMA-staged operands.
//   * A causal ConvTranspose1d(k = 2r, stride r) is the same kernel with 2 taps and N' = r*Cout "phase" channels;
//     the [T, r*Cout] result IS the [T*r, Cout] upsampled sequence (pixel shuffle is a reinterpretation).
//   * Epilogue fuses bias, residual add, and the NEXT layer's SnakeBeta (x + sin^2(a x) / (b + eps)), writing the raw
//     and/or the activated tensor, so no element-wise kernel exists in the stack.
// conv_out (96 -> 1 channel) + clamp is a small dedicated kernel.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "../../include/fq3_engine.h"
#include "fq3_gemm.cuh"

namespace {

thread_local char g_cerr[512] = "";
int cfail(int code, const char* msg, const char* extra = "") {
  snprintf(g_cerr, sizeof(g_cerr), "%s%s", msg, extra);
  return code;
}
#define CCK(call)                                                                  \
  do {                                                                             \
    cudaError_t _e = (call);                                                       \
    if (_e != cudaSuccess) return cfail(FQ3_ERR_CUDA, #call " failed: ", cudaGetErrorString(_e)); \
  } while (0)

using namespace fq3gemm;

// the caller's current device is restored when an entry point returns (single-process multi-GPU hosts, torch)
struct CodecDevGuard {
  int prev = -1, dev;
  explicit CodecDevGuard(int d) : dev(d) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) cudaSetDevice(dev);
  }
  ~CodecDevGuard() {
    if (prev >= 0 && prev != dev) cudaSetDevice(prev);
  }
};

// final causal conv7 (C -> 1) over activated input + clamp to [-1, 1]; one thread per output sample
__global__ void conv_out_kernel(const __nv_bfloat16* __restrict__ X, const float* __restrict__ W, float bias, int T,
                                int C, int taps, float* __restrict__ out, int x_row0, int x_rows) {
  pdl_launch();
  pdl_wait();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  X += (size_t)blockIdx.y * x_rows * C;  // blockIdx.y = sequence of the batch; its input has x_row0 history rows in front
  out += (size_t)blockIdx.y * T;
  float s = bias;
  for (int k = 0; k < taps; ++k) {
    const int tt = x_row0 + t - (taps - 1 - k);
    if (tt < 0) continue;
    const __nv_bfloat162* x = reinterpret_cast<const __nv_bfloat162*>(X + (size_t)tt * C);
    const float* w = W + (size_t)k * C;
    for (int c = 0; c < C / 2; ++c) {
      const __nv_bfloat162 v = x[c];
      s = fmaf(__bfloat162float(v.x), w[2 * c], s);
      s = fmaf(__bfloat162float(v.y), w[2 * c + 1], s);
    }
  }
  out[t] = fminf(1.f, fmaxf(-1.f, s));
}


// ============================================================================================================
// Front end of the decoder (everything of `speech_tokenizer.decode` before conv_in): RVQ code embedding mean ->
// sliding-window pre-transformer -> 2 x (ConvTranspose k=s + ConvNeXt).  Dense layers run on the same implicit-GEMM
// kernel as the stack (taps = 1; fused bias / layer-scale / residual / SwiGLU / GELU epilogues); the kernels below are
// the row-wise pieces between them.  All activations bf16 channels-last [batch * T][C]; roundings where the torch
// bf16 modules materialise a tensor.
// ============================================================================================================
namespace fe {

__device__ __forceinline__ float rb(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// x[row][:] = mean_q emb[q * codebook + codes[row][q]][:]      one block per (batch, t) row
__global__ void embed_mean_kernel(const long long* __restrict__ codes, const __nv_bfloat16* __restrict__ emb, int Q,
                                  int codebook, int H, __nv_bfloat16* __restrict__ X) {
  const size_t row = blockIdx.x;
  __shared__ long long ids[64];
  fq3gemm::pdl_launch();
  fq3gemm::pdl_wait();
  if ((int)threadIdx.x < Q) {
    long long c = codes[row * Q + threadIdx.x];
    c = c < 0 ? 0 : (c >= codebook ? codebook - 1 : c);
    ids[threadIdx.x] = (long long)threadIdx.x * codebook + c;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < H; k += blockDim.x) {
    float s = 0.f;
    for (int q = 0; q < Q; ++q) s += __bfloat162float(emb[(size_t)ids[q] * H + k]);
    X[row * H + k] = __float2bfloat16_rn(s / (float)Q);
  }
}

// one block (256 threads) per row: Y = w * rnd(x * rsqrt(mean(x^2) + eps))      H <= 2048
__global__ void rmsnorm_rows_kernel(const __nv_bfloat16* __restrict__ X, const float* __restrict__ w, int H, float eps,
                                    __nv_bfloat16* __restrict__ Y) {
  __shared__ float red[8];
  fq3gemm::pdl_launch();
  fq3gemm::pdl_wait();
  const size_t row = blockIdx.x;
  const int tid = threadIdx.x;
  float v[8];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int k = tid + i * 256;
    v[i] = k < H ? __bfloat162float(X[row * H + k]) : 0.f;
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
    if (k < H) Y[row * H + k] = __float2bfloat16_rn(rb(w[k]) * rb(v[i] * r));
  }
}

// RoPE in place on the q and k thirds of QKV [rows][3H]; one warp per (row, head, q|k); position = row % T.
// hd <= 128, rotate_half convention: o[e] = x[e] cos - x[e + hd/2] sin, o[e + hd/2] = x[e + hd/2] cos + x[e] sin
__global__ void rope_qk_kernel(__nv_bfloat16* __restrict__ QKV, int rows, int T, int nh, int hd,
                               const float* __restrict__ inv_freq, const int* __restrict__ pos0) {
  fq3gemm::pdl_launch();
  fq3gemm::pdl_wait();
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (gw >= rows * nh * 2) return;
  const int row = gw / (nh * 2), r = gw % (nh * 2), which = r / nh, h = r % nh;
  const int H = nh * hd, half = hd >> 1;
  __nv_bfloat16* p = QKV + (size_t)row * 3 * H + (size_t)which * H + (size_t)h * hd;
  const float pos = (float)((row % T) + (pos0 ? pos0[row / T] : 0));   // streaming: frames this sequence has seen before
  for (int e = lane; e < half; e += 32) {
    const float fr = pos * inv_freq[e];
    const float cs = rb(cosf(fr)), sn = rb(sinf(fr));
    const float a = __bfloat162float(p[e]), b = __bfloat162float(p[e + half]);
    p[e] = __float2bfloat16_rn(rb(a * cs) + rb(-b * sn));
    p[e + half] = __float2bfloat16_rn(rb(b * cs) + rb(a * sn));
  }
}

// causal sliding-window attention (keys j in (i - W, i]) of one head; block = 8 queries (one warp each).
// QKV [rows][3H] (RoPE applied), OUT [rows][H].  fp32 scores / softmax / P.V.
// Streaming: every sequence's QKV block has x_rows = row0 + T rows, the first row0 of them the cached (k, v) rows of
// earlier chunks, of which only the last valid[b] exist yet.
template <int HD>
__global__ void __launch_bounds__(256) swa_kernel(const __nv_bfloat16* __restrict__ QKV, int T, int nh, int W,
                                                  __nv_bfloat16* __restrict__ OUT, int x_rows, int row0,
                                                  const int* __restrict__ valid) {
  extern __shared__ float fsm[];
  fq3gemm::pdl_launch();
  fq3gemm::pdl_wait();
  const int Wpad = (W + 31) & ~31;
  float* sc = fsm;                  // [8][Wpad]
  float* qs = fsm + 8 * Wpad;       // [8][HD]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.y, b = blockIdx.z;
  const int i = blockIdx.x * 8 + warp;
  if (i >= T) return;
  const int H = nh * HD;
  const size_t ld = 3 * (size_t)H;
  const __nv_bfloat16* base = QKV + (size_t)b * x_rows * ld;
  const int ie = row0 + i;                                   // row of query i inside the sequence's block
  for (int e = lane; e < HD; e += 32) qs[warp * HD + e] = __bfloat162float(base[(size_t)ie * ld + h * HD + e]);
  __syncwarp();
  const int lo = max(row0 - (valid ? valid[b] : row0), ie - W + 1);
  const int nk = ie - lo + 1;
  const float scale = rsqrtf((float)HD);
  float* my = sc + warp * Wpad;
  const float* q = qs + warp * HD;
  float mx = -INFINITY;
  for (int jj = lane; jj < nk; jj += 32) {
    const uint4* kr = reinterpret_cast<const uint4*>(base + (size_t)(lo + jj) * ld + H + h * HD);
    float d = 0.f;
#pragma unroll
    for (int c = 0; c < HD / 8; ++c) {
      const uint4 w = __ldg(kr + c);
      const float* qq = q + c * 8;
      d = fmaf(qq[0], __uint_as_float(w.x << 16), d); d = fmaf(qq[1], __uint_as_float(w.x & 0xffff0000u), d);
      d = fmaf(qq[2], __uint_as_float(w.y << 16), d); d = fmaf(qq[3], __uint_as_float(w.y & 0xffff0000u), d);
      d = fmaf(qq[4], __uint_as_float(w.z << 16), d); d = fmaf(qq[5], __uint_as_float(w.z & 0xffff0000u), d);
      d = fmaf(qq[6], __uint_as_float(w.w << 16), d); d = fmaf(qq[7], __uint_as_float(w.w & 0xffff0000u), d);
    }
    d *= scale;
    my[jj] = d;
    mx = fmaxf(mx, d);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int jj = lane; jj < nk; jj += 32) {
    const float e = expf(my[jj] - mx);
    my[jj] = e;
    sum += e;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  __syncwarp();
  const float inv = 1.0f / sum;
  constexpr int EPL = HD / 32;      // dims per lane: [EPL * lane, EPL * lane + EPL)
  float acc[EPL];
#pragma unroll
  for (int e = 0; e < EPL; ++e) acc[e] = 0.f;
  for (int jj = 0; jj < nk; ++jj) {
    const float p = my[jj] * inv;
    const __nv_bfloat16* vr = base + (size_t)(lo + jj) * ld + 2 * H + h * HD + EPL * lane;
#pragma unroll
    for (int e = 0; e < EPL; ++e) acc[e] = fmaf(p, __bfloat162float(vr[e]), acc[e]);
  }
  __nv_bfloat16* o = OUT + ((size_t)b * T + i) * H + h * HD + EPL * lane;
#pragma unroll
  for (int e = 0; e < EPL; ++e) o[e] = __float2bfloat16_rn(acc[e]);
}

// ConvNeXt head: depthwise causal conv7 (+bias, rounded to bf16 like the conv module's output) followed by
// LayerNorm(C) with affine parameters.  One block (256 threads) per (batch, t) row; C <= 2048.
__global__ void dwconv_ln_kernel(const __nv_bfloat16* __restrict__ X, int T, int C, const float* __restrict__ w /*[C][7]*/,
                                 const float* __restrict__ bias, const float* __restrict__ lnw, const float* __restrict__ lnb,
                                 float eps, __nv_bfloat16* __restrict__ Y, int x_row0, int x_rows) {
  __shared__ float red[2][8];
  fq3gemm::pdl_launch();
  fq3gemm::pdl_wait();
  const size_t row = blockIdx.x;
  const int t = (int)(row % T) + x_row0;                                  // row inside the sequence's input block
  const size_t xrow = (row / T) * (size_t)x_rows + t;
  const int tid = threadIdx.x;
  float v[8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = tid + i * 256;
    v[i] = 0.f;
    if (c < C) {
      float a = rb(bias[c]);
#pragma unroll
      for (int k = 0; k < 7; ++k) {
        const int tt = t - 6 + k;
        if (tt >= 0) a = fmaf(rb(w[c * 7 + k]), __bfloat162float(X[(xrow - (size_t)(6 - k)) * C + c]), a);
      }
      v[i] = rb(a);
      s += v[i];
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((tid & 31) == 0) red[0][tid >> 5] = s;
  __syncthreads();
  float mean = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) mean += red[0][i];
  mean /= (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = tid + i * 256;
    if (c < C) q += (v[i] - mean) * (v[i] - mean);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  if ((tid & 31) == 0) red[1][tid >> 5] = q;
  __syncthreads();
  float var = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) var += red[1][i];
  const float r = 1.0f / sqrtf(var / (float)C + eps);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = tid + i * 256;
    if (c < C) Y[row * C + c] = __float2bfloat16_rn((v[i] - mean) * r * rb(lnw[c]) + rb(lnb[c]));
  }
}

}  // namespace fe

struct FeLayer {
  float *ln1 = nullptr, *ln2 = nullptr, *s1 = nullptr, *s2 = nullptr;
  __nv_bfloat16 *qkv = nullptr, *o = nullptr, *gu = nullptr, *down = nullptr;
};
struct FeUp {
  int r = 2;
  __nv_bfloat16 *ct = nullptr, *pw1 = nullptr, *pw2 = nullptr;
  float *ct_b = nullptr, *dw_w = nullptr, *dw_b = nullptr, *ln_w = nullptr, *ln_b = nullptr, *pw1_b = nullptr,
        *pw2_b = nullptr, *gamma = nullptr;
};
struct FrontEnd {
  bool ready = false;
  int Q = 16, codebook = 2048, H = 1024, I = 3072, nh = 16, L = 8, window = 72;
  float eps = 1e-5f, theta = 10000.f;
  __nv_bfloat16* emb = nullptr;
  float *norm = nullptr, *inv_freq = nullptr;
  std::vector<FeLayer> layers;
  std::vector<FeUp> ups;
  size_t cap_rows = 0;
  __nv_bfloat16* buf[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  double flops_per_frame = 0;
};

struct Layer {
  int Cin, N, taps, dil, bias_mod, act_mod;  // act_mod 0 => no activated output
  bool write_raw, residual;
  int upsample;                              // r for ConvTranspose-as-conv (T_out = T*r, channels N/r), else 1
  __nv_bfloat16* W = nullptr;
  float *bias = nullptr, *ea = nullptr, *ib = nullptr;
};

}  // namespace

struct fq3_codec {
  int dev = 0;
  int hidden = 0, decoder_dim = 0, n_blocks = 0;
  int rates[8];
  std::vector<Layer> layers;
  float* w_out = nullptr;
  float b_out = 0.f;
  int c_out = 0;
  // scratch (grown on demand)
  size_t cap = 0;
  __nv_bfloat16 *buf[4] = {nullptr, nullptr, nullptr, nullptr};
  int64_t launches = 0;
  double flops_per_frame = 0;
  std::vector<void*> owned;
  FrontEnd fe;
  // ---- stateful streaming (fq3_codec_stream_*): causal sites in execution order
  struct Site { int h, C; size_t off; };   // history rows / channels of the site's INPUT tensor, offset into a stream's tails
  std::vector<Site> sites;
  size_t tail_elems = 0;
  __nv_bfloat16* ext = nullptr;            // [batch][h + T][C] work buffer of the site being executed
  size_t ext_cap = 0;
  void** d_tailptr = nullptr;              // device copies of the per-call stream tables
  int* d_pos0 = nullptr;
  int* d_valid = nullptr;
  int tab_cap = 0;
};

struct fq3_codec_stream {
  fq3_codec* owner = nullptr;
  __nv_bfloat16* tails = nullptr;          // history rows of every causal site (zero = before the stream started)
  long long frames = 0;                    // code frames decoded so far
};

extern "C" int fq3_codec_create(const int32_t* geom, int32_t n_geom, fq3_codec** out) {
  // geom = {device, hidden_size, decoder_dim, n_blocks, rate_0 .. rate_{n-1}}
  if (!geom || !out || n_geom < 5) return cfail(FQ3_ERR_INVALID, "bad codec geometry");
  fq3_codec* c = new fq3_codec();
  c->dev = geom[0]; c->hidden = geom[1]; c->decoder_dim = geom[2]; c->n_blocks = geom[3];
  if (c->n_blocks < 1 || c->n_blocks > 8 || n_geom < 4 + c->n_blocks) { delete c; return cfail(FQ3_ERR_INVALID, "bad codec geometry"); }
  for (int i = 0; i < c->n_blocks; ++i) c->rates[i] = geom[4 + i];
  if (c->hidden % 32 || c->decoder_dim % (32 << c->n_blocks)) { delete c; return cfail(FQ3_ERR_INVALID, "codec channels must be multiples of 32 at every level"); }
  *out = c;
  return 0;
}

extern "C" void fq3_codec_destroy(fq3_codec* c) {
  if (!c) return;
  CodecDevGuard dev_guard(c->dev);
  for (void* p : c->owned) cudaFree(p);
  for (auto* b : c->buf) if (b) cudaFree(b);
  for (auto* b : c->fe.buf) if (b) cudaFree(b);
  if (c->ext) cudaFree(c->ext);
  if (c->d_tailptr) { cudaFree(c->d_tailptr); cudaFree(c->d_pos0); cudaFree(c->d_valid); }
  delete c;
}

// tensors (all float32 on device, PyTorch layouts; the engine converts / rearranges):
//   conv_in.w [D,H,7] conv_in.b [D]
//   b{i}.act.a b{i}.act.b [Cin]      b{i}.up.w [Cin,Cout,2r] b{i}.up.b [Cout]
//   b{i}.r{j}.a1.a .a1.b [C]  .c1.w [C,C,7] .c1.b [C]  .a2.a .a2.b [C]  .c2.w [C,C,1] .c2.b [C]
//   out.act.a out.act.b [C]   out.w [1,C,7] out.b [1]
extern "C" int fq3_codec_load_weights(fq3_codec* c, const fq3_tensor* tensors, int32_t n, void* stream_) {
  if (!c || !tensors) return cfail(FQ3_ERR_INVALID, "null argument");
  CodecDevGuard dev_guard(c->dev);
  cudaStream_t stream = (cudaStream_t)stream_;
  std::map<std::string, const fq3_tensor*> tm;
  for (int i = 0; i < n; ++i) tm[tensors[i].name] = &tensors[i];
  std::vector<std::vector<float>> keep;
  auto host = [&](const std::string& nm, int64_t numel, std::vector<float>& dst) -> int {
    auto it = tm.find(nm);
    if (it == tm.end()) return cfail(FQ3_ERR_INVALID, "missing codec tensor ", nm.c_str());
    if (it->second->numel != numel) return cfail(FQ3_ERR_INVALID, "bad numel for codec tensor ", nm.c_str());
    dst.resize(numel);
    CCK(cudaMemcpyAsync(dst.data(), it->second->dev_ptr, numel * sizeof(float), cudaMemcpyDeviceToHost, stream));
    CCK(cudaStreamSynchronize(stream));
    return 0;
  };
  auto up_f = [&](const std::vector<float>& v, float** d) -> int {
    CCK(cudaMalloc(d, v.size() * sizeof(float)));
    c->owned.push_back(*d);
    CCK(cudaMemcpyAsync(*d, v.data(), v.size() * sizeof(float), cudaMemcpyHostToDevice, stream));
    CCK(cudaStreamSynchronize(stream));
    return 0;
  };
  auto up_bf = [&](const std::vector<float>& v, __nv_bfloat16** d) -> int {
    std::vector<__nv_bfloat16> h(v.size());
    for (size_t i = 0; i < v.size(); ++i) h[i] = __float2bfloat16(v[i]);
    CCK(cudaMalloc(d, h.size() * 2));
    c->owned.push_back(*d);
    CCK(cudaMemcpyAsync(*d, h.data(), h.size() * 2, cudaMemcpyHostToDevice, stream));
    CCK(cudaStreamSynchronize(stream));
    return 0;
  };
  auto snake = [&](const std::string& pre, int C, float** ea, float** ib) -> int {
    std::vector<float> al, be;
    int rc;
    if ((rc = host(pre + ".a", C, al))) return rc;
    if ((rc = host(pre + ".b", C, be))) return rc;
    for (int i = 0; i < C; ++i) { al[i] = expf(al[i]); be[i] = 1.0f / (expf(be[i]) + 1e-9f); }
    if ((rc = up_f(al, ea))) return rc;
    return up_f(be, ib);
  };
  // causal conv weight [N, Cin, taps] (PyTorch) -> [N][taps][Cin]
  auto conv_w = [&](const std::string& nm, int N, int Cin, int taps, __nv_bfloat16** d) -> int {
    std::vector<float> w, r((size_t)N * taps * Cin);
    int rc;
    if ((rc = host(nm, (int64_t)N * Cin * taps, w))) return rc;
    for (int nn = 0; nn < N; ++nn)
      for (int ci = 0; ci < Cin; ++ci)
        for (int k = 0; k < taps; ++k) r[((size_t)nn * taps + k) * Cin + ci] = w[((size_t)nn * Cin + ci) * taps + k];
    return up_bf(r, d);
  };
  c->layers.clear();
  int rc;
  const int H = c->hidden, D = c->decoder_dim;
  double flops = 0;  // per input frame position of the stack (multiply by 4*T)
  double pos = 1.0;  // positions per stack-input position
  {  // conv_in: writes only the block-0 SnakeBeta-activated tensor
    Layer L{H, D, 7, 1, D, D, false, false, 1};
    if ((rc = conv_w("conv_in.w", D, H, 7, &L.W))) return rc;
    std::vector<float> b;
    if ((rc = host("conv_in.b", D, b))) return rc;
    if ((rc = up_f(b, &L.bias))) return rc;
    if ((rc = snake("b0.act", D, &L.ea, &L.ib))) return rc;
    c->layers.push_back(L);
    flops += 2.0 * D * H * 7 * pos;
  }
  int Cin = D;
  for (int bi = 0; bi < c->n_blocks; ++bi) {
    const int Cout = Cin / 2, r = c->rates[bi];
    const std::string p = "b" + std::to_string(bi);
    {  // ConvTranspose(k=2r, s=r) as a 2-tap conv with N' = r*Cout
      Layer L{Cin, r * Cout, 2, 1, Cout, Cout, true, false, r};
      std::vector<float> w, wr((size_t)r * Cout * 2 * Cin);
      if ((rc = host(p + ".up.w", (int64_t)Cin * Cout * 2 * r, w))) return rc;
      for (int j = 0; j < r; ++j)
        for (int co = 0; co < Cout; ++co)
          for (int ci = 0; ci < Cin; ++ci) {
            const size_t nrow = (size_t)j * Cout + co;
            wr[(nrow * 2 + 0) * Cin + ci] = w[((size_t)ci * Cout + co) * 2 * r + j + r];  // tap 0 <-> x[q-1]
            wr[(nrow * 2 + 1) * Cin + ci] = w[((size_t)ci * Cout + co) * 2 * r + j];      // tap 1 <-> x[q]
          }
      if ((rc = up_bf(wr, &L.W))) return rc;
      std::vector<float> b;
      if ((rc = host(p + ".up.b", Cout, b))) return rc;
      if ((rc = up_f(b, &L.bias))) return rc;
      if ((rc = snake(p + ".r0.a1", Cout, &L.ea, &L.ib))) return rc;
      c->layers.push_back(L);
      flops += 2.0 * r * Cout * 2 * Cin * pos;
      pos *= r;
    }
    static const int dils[3] = {1, 3, 9};
    for (int j = 0; j < 3; ++j) {
      const std::string q = p + ".r" + std::to_string(j);
      {  // conv7(dil) on act1(x) -> act2 fused
        Layer L{Cout, Cout, 7, dils[j], Cout, Cout, false, false, 1};
        if ((rc = conv_w(q + ".c1.w", Cout, Cout, 7, &L.W))) return rc;
        std::vector<float> b;
        if ((rc = host(q + ".c1.b", Cout, b))) return rc;
        if ((rc = up_f(b, &L.bias))) return rc;
        if ((rc = snake(q + ".a2", Cout, &L.ea, &L.ib))) return rc;
        c->layers.push_back(L);
      }
      {  // conv1 + residual -> raw (next residual) + the next consumer's SnakeBeta
        const bool last = j == 2;
        Layer L{Cout, Cout, 1, 1, Cout, Cout, !last, true, 1};
        if ((rc = conv_w(q + ".c2.w", Cout, Cout, 1, &L.W))) return rc;
        std::vector<float> b;
        if ((rc = host(q + ".c2.b", Cout, b))) return rc;
        if ((rc = up_f(b, &L.bias))) return rc;
        const std::string nxt = !last ? p + ".r" + std::to_string(j + 1) + ".a1"
                                      : (bi + 1 < c->n_blocks ? "b" + std::to_string(bi + 1) + ".act" : std::string("out.act"));
        if ((rc = snake(nxt, Cout, &L.ea, &L.ib))) return rc;
        c->layers.push_back(L);
      }
      flops += 2.0 * Cout * Cout * 8 * pos;
    }
    Cin = Cout;
  }
  {
    std::vector<float> w, wr((size_t)7 * Cin), b;
    if ((rc = host("out.w", (int64_t)Cin * 7, w))) return rc;
    for (int ci = 0; ci < Cin; ++ci)
      for (int k = 0; k < 7; ++k) wr[(size_t)k * Cin + ci] = w[(size_t)ci * 7 + k];
    if ((rc = up_f(wr, &c->w_out))) return rc;
    if ((rc = host("out.b", 1, b))) return rc;
    c->b_out = b[0];
    c->c_out = Cin;
    flops += 2.0 * Cin * 7 * pos;
  }
  c->flops_per_frame = flops;
  return 0;
}

static int launch_conv(fq3_codec* c, const Layer& L, const __nv_bfloat16* X, const __nv_bfloat16* R, __nv_bfloat16* Yraw,
                       __nv_bfloat16* Yact, int T, int batch, cudaStream_t stream, int x_row0, int x_rows) {
  ConvArgs a;
  a.X = X; a.W = L.W; a.bias = L.bias; a.R = R; a.Yraw = Yraw; a.Yact = Yact; a.ea = L.ea; a.ib = L.ib;
  a.T = T; a.Cin = L.Cin; a.N = L.N; a.taps = L.taps; a.dil = L.dil; a.bias_mod = L.bias_mod; a.act_mod = L.act_mod;
  a.mode = 0;
  a.scale = nullptr; a.scale_mod = 1;
  a.x_row0 = x_row0; a.x_rows = x_rows;
  a.batch = batch;
  c->launches++;
  if (const char* err = gemm(a, stream)) return cfail(FQ3_ERR_CUDA, "codec conv GEMM: ", err);
  return 0;
}

// ------------------------------------------------------------------------------------------------------------
// front end weights
// ------------------------------------------------------------------------------------------------------------
// dst[(n * dmul + dadd) * K + k] = bf16(src[off + n * sn + k * sk])   (weight repacking on device)
static __global__ void cast_strided_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long N,
                                           long long K, long long sn, long long sk, long long off, int dmul, int dadd) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * K) return;
  const long long n = i / K, k = i - n * K;
  dst[(n * dmul + dadd) * K + k] = __float2bfloat16_rn(src[off + n * sn + k * sk]);
}

/* geom = {Q, codebook_size, hidden, intermediate, n_heads, n_layers, sliding_window, n_up, ratio_0 ..};
 * fgeom = {rms_norm_eps, rope_theta}.  Tensors (float32 on device, PyTorch layouts):
 *   fe.embed [Q*codebook, H]   fe.norm [H]
 *   fe.l{i}.ln1 .ln2 .s1 .s2 [H]   .q .k .v .o [H,H]   .gate .up [I,H]   .down [H,I]
 *   fe.u{i}.ct.w [H,H,r] .ct.b [H]  .dw.w [H,1,7] .dw.b [H]  .ln.w .ln.b [H]  .pw1.w [4H,H] .pw1.b [4H]  .pw2.w [H,4H]
 *   .pw2.b [H]  .gamma [H] */
extern "C" int fq3_codec_load_frontend(fq3_codec* c, const int32_t* geom, int32_t n_geom, const float* fgeom,
                                       int32_t n_fgeom, const fq3_tensor* tensors, int32_t n, void* stream_) {
  if (!c || !geom || !fgeom || !tensors || n_geom < 8 || n_fgeom < 2) return cfail(FQ3_ERR_INVALID, "null argument");
  CodecDevGuard dev_guard(c->dev);
  cudaStream_t stream = (cudaStream_t)stream_;
  FrontEnd& f = c->fe;
  f.ready = false;
  f.Q = geom[0]; f.codebook = geom[1]; f.H = geom[2]; f.I = geom[3]; f.nh = geom[4]; f.L = geom[5]; f.window = geom[6];
  const int n_up = geom[7];
  if (n_geom < 8 + n_up) return cfail(FQ3_ERR_INVALID, "bad front-end geometry");
  f.eps = fgeom[0]; f.theta = fgeom[1];
  const int H = f.H, I = f.I;
  if (H != c->hidden) return cfail(FQ3_ERR_INVALID, "front-end hidden size differs from the stack's");
  const int hd = f.nh > 0 ? H / f.nh : 0;
  if (f.Q < 1 || f.Q > 64 || H % 64 || H > 2048 || I % 32 || f.nh < 1 || hd * f.nh != H || (hd != 64 && hd != 128) ||
      f.window < 1 || f.L < 0 || n_up < 0)
    return cfail(FQ3_ERR_INVALID, "front-end geometry unsupported (hidden % 64, head_dim 64/128, Q <= 64)");
  std::map<std::string, const fq3_tensor*> tm;
  for (int i = 0; i < n; ++i) tm[tensors[i].name] = &tensors[i];
  auto find = [&](const std::string& nm, int64_t numel, const float** p) -> int {
    auto it = tm.find(nm);
    if (it == tm.end()) return cfail(FQ3_ERR_INVALID, "missing codec tensor ", nm.c_str());
    if (it->second->numel != numel) return cfail(FQ3_ERR_INVALID, "bad numel for codec tensor ", nm.c_str());
    *p = (const float*)it->second->dev_ptr;
    return 0;
  };
  auto vec = [&](const std::string& nm, int64_t numel, float** d) -> int {
    const float* src;
    int rc = find(nm, numel, &src);
    if (rc) return rc;
    CCK(cudaMalloc(d, numel * sizeof(float)));
    c->owned.push_back(*d);
    CCK(cudaMemcpyAsync(*d, src, numel * sizeof(float), cudaMemcpyDeviceToDevice, stream));
    return 0;
  };
  auto alloc_bf = [&](int64_t numel, __nv_bfloat16** d) -> int {
    CCK(cudaMalloc(d, numel * 2));
    c->owned.push_back(*d);
    return 0;
  };
  auto cast = [&](const std::string& nm, int64_t N, int64_t K, int64_t sn, int64_t sk, int64_t off, int dmul, int dadd,
                  int64_t src_numel, __nv_bfloat16* dst) -> int {
    const float* src;
    int rc = find(nm, src_numel, &src);
    if (rc) return rc;
    const long long tot = N * K;
    cast_strided_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(src, dst, N, K, sn, sk, off, dmul, dadd);
    CCK(cudaGetLastError());
    return 0;
  };
  int rc;
  if ((rc = alloc_bf((int64_t)f.Q * f.codebook * H, &f.emb))) return rc;
  if ((rc = cast("fe.embed", (int64_t)f.Q * f.codebook, H, H, 1, 0, 1, 0, (int64_t)f.Q * f.codebook * H, f.emb))) return rc;
  if ((rc = vec("fe.norm", H, &f.norm))) return rc;
  {
    std::vector<float> inv(hd / 2);
    for (int i = 0; i < hd / 2; ++i) inv[i] = 1.0f / powf(f.theta, (float)(2 * i) / (float)hd);
    CCK(cudaMalloc(&f.inv_freq, inv.size() * sizeof(float)));
    c->owned.push_back(f.inv_freq);
    CCK(cudaMemcpyAsync(f.inv_freq, inv.data(), inv.size() * sizeof(float), cudaMemcpyHostToDevice, stream));
    CCK(cudaStreamSynchronize(stream));
  }
  f.layers.assign(f.L, FeLayer());
  double flops = 0;
  for (int l = 0; l < f.L; ++l) {
    FeLayer& y = f.layers[l];
    const std::string p = "fe.l" + std::to_string(l);
    if ((rc = vec(p + ".ln1", H, &y.ln1)) || (rc = vec(p + ".ln2", H, &y.ln2)) || (rc = vec(p + ".s1", H, &y.s1)) ||
        (rc = vec(p + ".s2", H, &y.s2)))
      return rc;
    if ((rc = alloc_bf((int64_t)3 * H * H, &y.qkv)) || (rc = alloc_bf((int64_t)H * H, &y.o)) ||
        (rc = alloc_bf((int64_t)2 * I * H, &y.gu)) || (rc = alloc_bf((int64_t)H * I, &y.down)))
      return rc;
    const char* qkvn[3] = {".q", ".k", ".v"};
    for (int j = 0; j < 3; ++j)
      if ((rc = cast(p + qkvn[j], H, H, H, 1, 0, 1, 0, (int64_t)H * H, y.qkv + (size_t)j * H * H))) return rc;
    if ((rc = cast(p + ".o", H, H, H, 1, 0, 1, 0, (int64_t)H * H, y.o))) return rc;
    if ((rc = cast(p + ".gate", I, H, H, 1, 0, 2, 0, (int64_t)I * H, y.gu))) return rc;   // interleaved gate / up rows
    if ((rc = cast(p + ".up", I, H, H, 1, 0, 2, 1, (int64_t)I * H, y.gu))) return rc;
    if ((rc = cast(p + ".down", H, I, I, 1, 0, 1, 0, (int64_t)H * I, y.down))) return rc;
    flops += 2.0 * (4.0 * H * H + 3.0 * H * I);
  }
  f.ups.assign(n_up, FeUp());
  double pos = 1.0;
  for (int u = 0; u < n_up; ++u) {
    FeUp& y = f.ups[u];
    y.r = geom[8 + u];
    if (y.r < 1 || y.r > 8) return cfail(FQ3_ERR_INVALID, "bad upsampling ratio");
    const int r = y.r;
    const std::string p = "fe.u" + std::to_string(u);
    if ((rc = alloc_bf((int64_t)r * H * H, &y.ct)) || (rc = alloc_bf((int64_t)4 * H * H, &y.pw1)) ||
        (rc = alloc_bf((int64_t)4 * H * H, &y.pw2)))
      return rc;
    // ConvTranspose1d(k = s = r): phase j, output channel co  <-  row j*H + co ;  W'[row][ci] = w[ci][co][j]
    for (int j = 0; j < r; ++j)
      if ((rc = cast(p + ".ct.w", H, H, r, (int64_t)H * r, j, 1, j * H, (int64_t)H * H * r, y.ct))) return rc;
    if ((rc = cast(p + ".pw1.w", 4 * H, H, H, 1, 0, 1, 0, (int64_t)4 * H * H, y.pw1))) return rc;
    if ((rc = cast(p + ".pw2.w", H, 4 * H, 4 * H, 1, 0, 1, 0, (int64_t)4 * H * H, y.pw2))) return rc;
    if ((rc = vec(p + ".ct.b", H, &y.ct_b)) || (rc = vec(p + ".dw.w", (int64_t)H * 7, &y.dw_w)) ||
        (rc = vec(p + ".dw.b", H, &y.dw_b)) || (rc = vec(p + ".ln.w", H, &y.ln_w)) || (rc = vec(p + ".ln.b", H, &y.ln_b)) ||
        (rc = vec(p + ".pw1.b", 4 * H, &y.pw1_b)) || (rc = vec(p + ".pw2.b", H, &y.pw2_b)) ||
        (rc = vec(p + ".gamma", H, &y.gamma)))
      return rc;
    flops += 2.0 * r * H * H * pos;
    pos *= r;
    flops += 2.0 * 8.0 * H * H * pos;
  }
  CCK(cudaStreamSynchronize(stream));
  f.flops_per_frame = flops;
  CCK(cudaFuncSetAttribute(fe::swa_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
  CCK(cudaFuncSetAttribute(fe::swa_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
  f.ready = true;
  return 0;
}

static int fe_gemm(fq3_codec* c, const __nv_bfloat16* X, const __nv_bfloat16* W, const float* bias, const float* scale,
                   const __nv_bfloat16* R, __nv_bfloat16* Y, int rows, int K, int N, int bias_mod, int mode,
                   cudaStream_t stream) {
  ConvArgs a;
  memset(&a, 0, sizeof(a));
  a.X = X; a.W = W; a.bias = bias; a.R = R; a.Yraw = Y; a.T = rows; a.Cin = K; a.N = N; a.taps = 1; a.dil = 1;
  a.bias_mod = bias_mod; a.act_mod = 1; a.mode = mode; a.scale = scale; a.scale_mod = N; a.batch = 1;
  c->launches++;
  if (const char* err = gemm(a, stream)) return cfail(FQ3_ERR_CUDA, "codec front-end GEMM: ", err);
  return 0;
}


// ------------------------------------------------------------------------------------------------------------
// Stateful streaming decode (SURVEY 8(f) item 2): instead of re-decoding a window of old frames for every chunk
// (the reference's Phase-1 O(n^2) re-decode and 25-frame Phase-2 context, model.py:1085-1135), every causal layer
// keeps the tail of its own input -- (k-1)*dilation rows for a causal conv, 1 row for a transposed conv, the last
// window-1 (k, v) rows for the sliding-window attention -- and a chunk costs only its own frames.  Each output row is
// computed by exactly the arithmetic of a one-shot decode of the whole sequence (the model is causal), so the PCM of a
// stream equals the non-streaming decode of the same codes.  The one-shot decode is the same forward (codec_forward)
// without history.
// ------------------------------------------------------------------------------------------------------------
static __global__ void ext_build_kernel(const __nv_bfloat16* const* __restrict__ tails, size_t off,
                                        const __nv_bfloat16* __restrict__ X, int h, int T, int C8,
                                        __nv_bfloat16* __restrict__ E) {
  // E[b][r][:] = r < h ? tail_b[r][:] : X[b][r - h][:]        (16-byte vectors; C8 = C / 8)
  fq3gemm::pdl_launch();
  fq3gemm::pdl_wait();
  const int b = blockIdx.y;
  const long long n = (long long)(h + T) * C8;
  const uint4* tb = reinterpret_cast<const uint4*>(tails[b] + off);
  const uint4* xb = reinterpret_cast<const uint4*>(X) + (size_t)b * T * C8;
  uint4* eb = reinterpret_cast<uint4*>(E) + (size_t)b * (h + T) * C8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / C8;
    eb[i] = r < h ? tb[i] : xb[i - (long long)h * C8];
  }
}
static __global__ void tail_save_kernel(__nv_bfloat16* const* __restrict__ tails, size_t off,
                                        const __nv_bfloat16* __restrict__ E, int h, int T, int C8) {
  // tail_b <- last h rows of E[b]
  fq3gemm::pdl_launch();
  fq3gemm::pdl_wait();
  const int b = blockIdx.y;
  const long long n = (long long)h * C8;
  uint4* tb = reinterpret_cast<uint4*>(tails[b] + off);
  const uint4* eb = reinterpret_cast<const uint4*>(E) + ((size_t)b * (h + T) + T) * C8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) tb[i] = eb[i];
}

static int stream_sites(fq3_codec* c) {
  if (!c->sites.empty()) return 0;
  const FrontEnd& f = c->fe;
  size_t off = 0;
  auto add = [&](int h, int C) { c->sites.push_back({h, C, off}); off += (size_t)h * C; };
  for (int l = 0; l < f.L; ++l) add(f.window - 1, 3 * f.H);
  for (size_t u = 0; u < f.ups.size(); ++u) add(6, f.H);
  for (const Layer& L : c->layers) add((L.taps - 1) * L.dil, L.Cin);   // pointwise layers: h = 0
  add(6, c->c_out);
  c->tail_elems = off;
  return 0;
}

// front-end and waveform-stack activations of `batch` sequences of T code frames (grown on demand)
static int reserve(fq3_codec* c, int batch, int T) {
  FrontEnd& f = c->fe;
  const size_t rows0 = (size_t)batch * T;
  size_t up = 1;
  for (auto& u : f.ups) up *= (size_t)u.r;
  const size_t rowsU = rows0 * up;
  if (rowsU > f.cap_rows) {
    for (auto*& b : f.buf) { if (b) cudaFree(b); b = nullptr; }
    const size_t wide = std::max(rows0 * (size_t)std::max(3 * f.H, f.I), rowsU * (size_t)4 * f.H);
    for (int i = 0; i < 5; ++i) CCK(cudaMalloc(&f.buf[i], (i == 3 ? wide : rowsU * (size_t)f.H) * 2));
    f.cap_rows = rowsU;
  }
  // waveform stack: largest tensor [T_final][C_final * 2] worth of bf16 at the widest level; every buffer sized for it
  size_t Tl = (size_t)T * up;
  int C = c->decoder_dim;
  size_t need = std::max(Tl * c->hidden, Tl * (size_t)C);
  for (int bi = 0; bi < c->n_blocks; ++bi) {
    Tl *= c->rates[bi];
    C /= 2;
    need = std::max(need, Tl * (size_t)C);
  }
  need *= (size_t)batch;
  if (need > c->cap) {
    for (auto*& b : c->buf) { if (b) cudaFree(b); b = nullptr; }
    for (auto*& b : c->buf) CCK(cudaMalloc(&b, need * 2));
    c->cap = need;
  }
  return 0;
}

/* The codec forward of both entry points: codes int64 [batch][T][Q] (device) -> PCM float32 [batch][T * total_upsample]
 * clamped to [-1, 1]; conv_out is skipped when pcm_out_dev is NULL.  history = true: every causal site reads the
 * streams' tails in front of its new rows, through the per-call tables (d_tailptr, d_pos0, d_valid) and c->ext that
 * fq3_codec_stream_decode has set up, and saves its new tail.  history = false: the one-shot decode, the same launches
 * without the history copies -- no site has rows in front, no sequence has earlier positions. */
static int codec_forward(fq3_codec* c, const int64_t* codes_dev, int batch, int T, float* pcm_out_dev, bool history,
                         cudaStream_t stream) {
  FrontEnd& f = c->fe;
  const int H = f.H, I = f.I, hd = H / f.nh;
  const int Wpad = (f.window + 31) & ~31;
  const size_t swa_smem = (size_t)(8 * Wpad + 8 * hd) * sizeof(float);
  if (swa_smem > 96 * 1024) return cfail(FQ3_ERR_INVALID, "sliding window too large");
  int rc;
  if ((rc = reserve(c, batch, T))) return rc;
  const int* pos0 = history ? c->d_pos0 : nullptr;
  const int* valid = history ? c->d_valid : nullptr;
  size_t site = 0;
  // input X [batch][Tn][C] of the next causal site with its h history rows in front -> c->ext [batch][h + Tn][C], the
  // streams' tails updated; X itself when h = 0
  auto with_history = [&](const __nv_bfloat16* X, int Tn, int& h) -> const __nv_bfloat16* {
    h = 0;
    if (!history) return X;
    const fq3_codec::Site& st = c->sites[site++];
    if (st.h == 0) return X;
    h = st.h;
    const int C8 = st.C / 8;
    const long long n = (long long)(st.h + Tn) * C8;
    dim3 g((unsigned)std::min<long long>((n + 255) / 256, 1024), batch);
    FQ3_LAUNCH((ext_build_kernel), g, 256, 0, stream, (const __nv_bfloat16* const*)c->d_tailptr, st.off, X, st.h, Tn, C8, c->ext);
    dim3 g2((unsigned)std::min<long long>(((long long)st.h * C8 + 255) / 256, 256), batch);
    FQ3_LAUNCH((tail_save_kernel), g2, 256, 0, stream, (__nv_bfloat16* const*)c->d_tailptr, st.off, c->ext, st.h, Tn, C8);
    c->launches += 2;
    return c->ext;
  };
  int h;
  // ---- front end
  __nv_bfloat16 *A = f.buf[0], *Bx = f.buf[1], *Cn = f.buf[2], *D = f.buf[3], *E = f.buf[4];
  const int R0 = batch * T;
  FQ3_LAUNCH((fe::embed_mean_kernel), R0, 256, 0, stream, (const long long*)codes_dev, f.emb, f.Q, f.codebook, H, A);
  c->launches++;
  for (int l = 0; l < f.L; ++l) {
    const FeLayer& y = f.layers[l];
    FQ3_LAUNCH((fe::rmsnorm_rows_kernel), R0, 256, 0, stream, A, y.ln1, H, f.eps, Cn);
    if ((rc = fe_gemm(c, Cn, y.qkv, nullptr, nullptr, nullptr, D, R0, H, 3 * H, 1, 0, stream))) return rc;
    {
      const long long warps = (long long)R0 * f.nh * 2;
      FQ3_LAUNCH((fe::rope_qk_kernel), (unsigned)((warps * 32 + 255) / 256), 256, 0, stream, D, R0, T, f.nh, hd, f.inv_freq, pos0);
    }
    const __nv_bfloat16* qkv = with_history(D, T, h);
    {
      dim3 g((T + 7) / 8, f.nh, batch);
      if (hd == 64) FQ3_LAUNCH((fe::swa_kernel<64>), g, 256, swa_smem, stream, qkv, T, f.nh, f.window, E, h + T, h, valid);
      else FQ3_LAUNCH((fe::swa_kernel<128>), g, 256, swa_smem, stream, qkv, T, f.nh, f.window, E, h + T, h, valid);
    }
    if ((rc = fe_gemm(c, E, y.o, nullptr, y.s1, A, Bx, R0, H, H, 1, 0, stream))) return rc;
    FQ3_LAUNCH((fe::rmsnorm_rows_kernel), R0, 256, 0, stream, Bx, y.ln2, H, f.eps, Cn);
    if ((rc = fe_gemm(c, Cn, y.gu, nullptr, nullptr, nullptr, D, R0, H, 2 * I, 1, 1, stream))) return rc;
    if ((rc = fe_gemm(c, D, y.down, nullptr, y.s2, Bx, A, R0, I, H, 1, 0, stream))) return rc;
    c->launches += 4;
  }
  FQ3_LAUNCH((fe::rmsnorm_rows_kernel), R0, 256, 0, stream, A, f.norm, H, f.eps, Cn);
  c->launches++;
  __nv_bfloat16* cur = Cn;
  int rows = R0, Ts = T;
  for (size_t u = 0; u < f.ups.size(); ++u) {
    const FeUp& y = f.ups[u];
    __nv_bfloat16* out = (cur == Cn) ? E : Cn;
    // ConvTranspose1d(k = s = r) as a GEMM onto r*H phase channels: [rows][r*H] IS [rows*r][H]
    if ((rc = fe_gemm(c, cur, y.ct, y.ct_b, nullptr, nullptr, A, rows, H, y.r * H, H, 0, stream))) return rc;
    rows *= y.r;
    Ts *= y.r;
    const __nv_bfloat16* xin = with_history(A, Ts, h);
    FQ3_LAUNCH((fe::dwconv_ln_kernel), rows, 256, 0, stream, xin, Ts, H, y.dw_w, y.dw_b, y.ln_w, y.ln_b, 1e-6f, Bx, h, h + Ts);
    c->launches++;
    if ((rc = fe_gemm(c, Bx, y.pw1, y.pw1_b, nullptr, nullptr, D, rows, H, 4 * H, 4 * H, 2, stream))) return rc;
    if ((rc = fe_gemm(c, D, y.pw2, y.pw2_b, y.gamma, A, out, rows, 4 * H, H, H, 0, stream))) return rc;
    cur = out;
  }
  CCK(cudaGetLastError());
  // ---- waveform stack
  size_t li = 0;
  auto conv = [&](const Layer& L, const __nv_bfloat16* X, const __nv_bfloat16* R, __nv_bfloat16* Yraw, __nv_bfloat16* Yact) -> int {
    const __nv_bfloat16* xin = with_history(X, Ts, h);
    return launch_conv(c, L, xin, R, Yraw, Yact, Ts, batch, stream, h, h + Ts);
  };
  // four ping-pong buffers.  `act` always holds the activated input of the next layer; the other three are free.
  __nv_bfloat16* act = c->buf[1];
  if ((rc = conv(c->layers[li++], cur, nullptr, nullptr, act))) return rc;
  for (int bi = 0; bi < c->n_blocks; ++bi) {
    __nv_bfloat16* fr[3];
    int k = 0;
    for (auto* b : c->buf)
      if (b != act) fr[k++] = b;
    __nv_bfloat16 *x = fr[0], *a1 = fr[1], *a2 = fr[2], *y = act;  // act is free once the up-conv has consumed it
    const Layer& U = c->layers[li++];
    if ((rc = conv(U, act, nullptr, x, a1))) return rc;  // raw -> x, SnakeBeta(raw) -> a1
    Ts *= U.upsample;
    for (int j = 0; j < 3; ++j) {
      const Layer& C1 = c->layers[li++];
      const Layer& C2 = c->layers[li++];
      if ((rc = conv(C1, a1, nullptr, nullptr, a2))) return rc;  // a2 = act2(conv7(a1))
      // y = conv1(a2) + x ; a1 <- SnakeBeta_next(y)   (conv7 has consumed a1, so it can be overwritten)
      if ((rc = conv(C2, a2, x, C2.write_raw ? y : nullptr, a1))) return rc;
      std::swap(x, y);
    }
    act = a1;
  }
  const __nv_bfloat16* xin = with_history(act, Ts, h);   // conv_out's history advances even when no PCM is wanted
  if (pcm_out_dev) {
    FQ3_LAUNCH((conv_out_kernel), dim3((Ts + 255) / 256, batch), 256, 0, stream, xin, c->w_out, c->b_out, Ts, c->c_out, 7, pcm_out_dev, h, h + Ts);
    c->launches++;
  }
  CCK(cudaGetLastError());
  return 0;
}

/* speech_tokenizer.decode (model.py:924,1093,1122) in one call: codes int64 [batch][T][Q] (device) -> PCM float32
 * [batch][T * total_upsample], clamped to [-1, 1].  `batch` windows of equal length share every launch. */
extern "C" int fq3_codec_decode_codes(fq3_codec* c, const int64_t* codes_dev, int32_t batch, int32_t T, float* pcm_out_dev,
                                      void* stream_) {
  if (!c || !codes_dev || !pcm_out_dev || T <= 0 || batch <= 0) return cfail(FQ3_ERR_INVALID, "null argument");
  if (c->layers.empty()) return cfail(FQ3_ERR_STATE, "codec weights not loaded");
  if (!c->fe.ready) return cfail(FQ3_ERR_STATE, "fq3_codec_load_frontend has not been called");
  CodecDevGuard dev_guard(c->dev);
  return codec_forward(c, codes_dev, batch, T, pcm_out_dev, false, (cudaStream_t)stream_);
}

extern "C" int fq3_codec_stream_create(fq3_codec* c, fq3_codec_stream** out) {
  if (!c || !out) return cfail(FQ3_ERR_INVALID, "null argument");
  if (c->layers.empty() || !c->fe.ready) return cfail(FQ3_ERR_STATE, "codec weights / front end not loaded");
  CodecDevGuard dev_guard(c->dev);
  stream_sites(c);
  fq3_codec_stream* s = new fq3_codec_stream();
  s->owner = c;
  if (cudaMalloc(&s->tails, c->tail_elems * 2) != cudaSuccess) { delete s; return cfail(FQ3_ERR_CUDA, "cudaMalloc of the stream state failed"); }
  if (cudaMemset(s->tails, 0, c->tail_elems * 2) != cudaSuccess) { cudaFree(s->tails); delete s; return cfail(FQ3_ERR_CUDA, "cudaMemset failed"); }
  *out = s;
  return 0;
}
extern "C" int fq3_codec_stream_reset(fq3_codec_stream* s, void* stream_) {
  if (!s) return cfail(FQ3_ERR_INVALID, "null argument");
  CodecDevGuard dev_guard(s->owner->dev);
  CCK(cudaMemsetAsync(s->tails, 0, s->owner->tail_elems * 2, (cudaStream_t)stream_));
  s->frames = 0;
  return 0;
}
extern "C" void fq3_codec_stream_destroy(fq3_codec_stream* s) {
  if (!s) return;
  CodecDevGuard dev_guard(s->owner->dev);
  cudaFree(s->tails);
  delete s;
}
extern "C" int64_t fq3_codec_stream_frames(fq3_codec_stream* s) { return s ? s->frames : 0; }
/* dst becomes a copy of src (state of every causal layer + position): a stream warmed once with a reference's frames
 * serves as the template of every later request with that reference (3.8 MB device-to-device, stream-ordered) */
extern "C" int fq3_codec_stream_copy(fq3_codec_stream* dst, fq3_codec_stream* src, void* stream_) {
  if (!dst || !src || dst->owner != src->owner) return cfail(FQ3_ERR_INVALID, "streams of different codecs");
  if (dst == src) return 0;
  CodecDevGuard dev_guard(src->owner->dev);
  CCK(cudaMemcpyAsync(dst->tails, src->tails, src->owner->tail_elems * 2, cudaMemcpyDeviceToDevice, (cudaStream_t)stream_));
  dst->frames = src->frames;
  return 0;
}

/* The next T code frames of n_streams streams (each with its own history) in one set of launches:
 * codes_dev int64 [n_streams][T][Q] -> pcm float32 [n_streams][T * total_upsample]; pcm_out_dev may be NULL (state
 * warm-up, e.g. the ICL reference frames: the waveform of the last stage is skipped, every state is updated). */
extern "C" int fq3_codec_stream_decode(fq3_codec* c, fq3_codec_stream* const* streams, int32_t n_streams,
                                       const int64_t* codes_dev, int32_t T, float* pcm_out_dev, void* stream_) {
  if (!c || !streams || !codes_dev || T <= 0 || n_streams <= 0) return cfail(FQ3_ERR_INVALID, "null argument");
  FrontEnd& f = c->fe;
  if (c->layers.empty() || !f.ready) return cfail(FQ3_ERR_STATE, "codec weights / front end not loaded");
  for (int b = 0; b < n_streams; ++b) {
    if (!streams[b] || streams[b]->owner != c) return cfail(FQ3_ERR_INVALID, "stream does not belong to this codec");
    for (int a = 0; a < b; ++a)
      if (streams[a] == streams[b]) return cfail(FQ3_ERR_INVALID, "stream listed twice");
  }
  CodecDevGuard dev_guard(c->dev);
  cudaStream_t stream = (cudaStream_t)stream_;
  stream_sites(c);
  const int batch = n_streams, W1 = f.window - 1;
  // ---- per-call stream tables
  if (batch > c->tab_cap) {
    if (c->d_tailptr) { cudaFree(c->d_tailptr); cudaFree(c->d_pos0); cudaFree(c->d_valid); }
    CCK(cudaMalloc(&c->d_tailptr, batch * sizeof(void*)));
    CCK(cudaMalloc(&c->d_pos0, batch * sizeof(int)));
    CCK(cudaMalloc(&c->d_valid, batch * sizeof(int)));
    c->tab_cap = batch;
  }
  {
    std::vector<void*> tp(batch);
    std::vector<int> p0(batch), vd(batch);
    for (int b = 0; b < batch; ++b) {
      tp[b] = streams[b]->tails;
      p0[b] = (int)streams[b]->frames;
      vd[b] = (int)std::min<long long>(streams[b]->frames, W1);
    }
    CCK(cudaMemcpyAsync(c->d_tailptr, tp.data(), batch * sizeof(void*), cudaMemcpyHostToDevice, stream));
    CCK(cudaMemcpyAsync(c->d_pos0, p0.data(), batch * sizeof(int), cudaMemcpyHostToDevice, stream));
    CCK(cudaMemcpyAsync(c->d_valid, vd.data(), batch * sizeof(int), cudaMemcpyHostToDevice, stream));
    // pageable sources: cudaMemcpyAsync returns once they have been staged, so the vectors may go out of scope here
  }
  // ---- c->ext: the largest site input with its history rows in front
  {
    size_t need = 0, Tl = T;
    size_t si = 0;
    for (int l = 0; l < f.L; ++l, ++si) need = std::max(need, (size_t)(c->sites[si].h + Tl) * c->sites[si].C);
    for (auto& u : f.ups) { Tl *= u.r; need = std::max(need, (size_t)(c->sites[si].h + Tl) * c->sites[si].C); ++si; }
    for (const Layer& L : c->layers) { need = std::max(need, (size_t)(c->sites[si].h + Tl) * c->sites[si].C); ++si; Tl *= L.upsample; }
    need = std::max(need, (size_t)(c->sites[si].h + Tl) * c->sites[si].C);
    need *= (size_t)batch;
    if (need > c->ext_cap) {
      if (c->ext) cudaFree(c->ext);
      c->ext = nullptr;
      CCK(cudaMalloc(&c->ext, need * 2));
      c->ext_cap = need;
    }
  }
  int rc;
  if ((rc = codec_forward(c, codes_dev, batch, T, pcm_out_dev, true, stream))) return rc;
  for (int b = 0; b < batch; ++b) streams[b]->frames += T;
  return 0;
}

extern "C" double fq3_codec_flops(fq3_codec* c, int32_t T4) { return c ? c->flops_per_frame * T4 : 0.0; }
/* front end FLOPs for T code frames (dense layers only) */
extern "C" double fq3_codec_frontend_flops(fq3_codec* c, int32_t T) { return c ? c->fe.flops_per_frame * T : 0.0; }
extern "C" int64_t fq3_codec_launch_count(fq3_codec* c) { return c ? c->launches : 0; }
extern "C" const char* fq3_codec_last_error(void) { return g_cerr; }
