// fq3_tempo.cu -- speaking-rate control: a pitch-preserving time-stretch (WSOLA, waveform-similarity overlap-add) of
// 24 kHz PCM that is already on the device, for any number of streams in one launch.  The algorithm is fixed exactly
// (DESIGN.md, "Speaking rate"; faster_qwen3_tts/tempo.py restates the counts, oracle/tempo_oracle.py the arithmetic):
//
//   x~ = H zeros, then the input (and, at flush only, zeros after its end).  Frame k has the nominal position
//   a_k = (k*H*q) >> 10 and, for k >= 1, the target t[n] = x~[p_{k-1} + H + n]; the candidates p = a_k + d, |d| <= D,
//   p >= 0, score c(p) = sum t[n] x~[p+n] / sqrt(eps + sum x~[p+n]^2); p_k = argmax, ties to the smallest |d|, then
//   the smaller p; p_0 = 0.  Overlap-add y~[kH + n] += w[n] x~[p_k + n] (the earlier frame's term first); y[m] = y~[m+H].
//
// A frame runs once every sample it can read exists, and output is released once no later frame can add to it, so the
// counts of a push are a function of the stream's totals alone: the host sizes every buffer before the launch and no
// value ever comes back.  The output depends on the input samples and the flush point only, never on how the input
// was split into pushes: a frame's reads and its reduction order are the same whichever push it runs in.
//
// One CTA per stream walks that stream's frames in order (p_k depends on p_{k-1}); the 2D+1 = 481 candidates of a
// frame are scored in parallel, one per thread, from a shared-memory copy of the searched span.  New samples are read
// in place from the caller's buffer; the per-stream device state holds the input tail later frames can still reach
// (< TCAP samples whatever the push length), the pending overlap, and p_{k-1}.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include <algorithm>
#include <vector>

#include "../../include/fq3_engine.h"

namespace {

constexpr int N = FQ3_TEMPO_WINDOW;        // 480 (20 ms): periodic Hann
constexpr int H = N / 2;                   // synthesis hop
constexpr int D = FQ3_TEMPO_SEARCH;        // 240: search half-width
constexpr int SPAN = 2 * D + N;            // samples a frame's candidates read
constexpr int TCAP = 2048;                 // retained input tail (the largest reach is 1680, at q = 4096)
constexpr int THREADS = 512;               // >= 2D + 1 candidates
constexpr float EPS = FQ3_TEMPO_EPS;
static_assert(THREADS >= 2 * D + 1, "one thread per candidate");

// device state of one stream: two tail buffers (ping-pong across calls), the pending overlap, p_{k-1}
constexpr size_t PENDING_OFF = 2 * TCAP;
constexpr size_t PPREV_OFF = PENDING_OFF + H;      // in floats; 8-byte aligned, holds one int64
constexpr size_t STATE_FLOATS = PPREV_OFF + 2;

thread_local char g_terr[256] = "";
int tfail(int code, const char* msg) {
  snprintf(g_terr, sizeof(g_terr), "%s", msg);
  return code;
}

struct DevGuard {
  int prev = -1, dev;
  explicit DevGuard(int d) : dev(d) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) cudaSetDevice(dev);
  }
  ~DevGuard() {
    if (prev >= 0 && prev != dev) cudaSetDevice(prev);
  }
};

int64_t nominal(int64_t k, int q) { return (k * H * q) >> 10; }

// frames that can run with L input samples (no flush): frame 0 needs x~[0, N); frame k >= 1 reads up to
// max(a_k, a_{k-1} + H) + D + N (exclusive), the farthest its candidates or its target (p_{k-1} <= a_{k-1} + D) reach
int64_t ready_frames(int64_t L, int q) {
  const int64_t lim = H + L;
  if (lim < N) return 0;
  const int64_t m = lim - D - N;       // frame k >= 1 runs iff a_k <= m and a_{k-1} <= m - H
  if (m - H < 0) return 1;
  const int64_t k1 = ((m + 1) * 1024 - 1) / ((int64_t)H * q);
  const int64_t k2 = ((m - H + 1) * 1024 - 1) / ((int64_t)H * q) + 1;
  return std::min(k1, k2) + 1;
}

// first x~ index any frame >= K can read
int64_t reach_lo(int64_t K, int q) {
  if (K == 0) return 0;
  return std::min(std::max<int64_t>(0, nominal(K, q) - D), std::max<int64_t>(0, nominal(K - 1, q) - D) + H);
}

struct Job {
  float* state;
  const float* in;     // new samples x[L0, L1)
  float* out;          // y[E0, E1)
  int32_t* pk;         // p_k of frames [K0, K1), or null
  long long L0, L1, ts0, ts1, K0, K1, E0, E1;
  int q, cur, flush;
};

__device__ __forceinline__ float xt(const Job& J, const float* tail, long long i) {
  // x~[i]: zeros in front, the retained tail, the new samples, zeros after the end (flush)
  if (i < H) return 0.f;
  const long long j = i - H;
  if (j < J.L0) return tail[j - J.ts0];
  if (j < J.L1) return J.in[j - J.L0];
  return 0.f;
}

struct Best {
  float s;
  int d, c;
};
__device__ __forceinline__ bool better(const Best& a, const Best& b) {
  return a.s > b.s || (a.s == b.s && (a.d < b.d || (a.d == b.d && a.c < b.c)));
}

__global__ void __launch_bounds__(THREADS) tempo_kernel(const Job* __restrict__ jobs) {
  const Job J = jobs[blockIdx.x];
  __shared__ float win[SPAN], tgt[N], pend[H], hann[N];
  __shared__ Best part[THREADS / 32];
  __shared__ long long best_p;
  const int tid = threadIdx.x;
  const float* tail = J.state + (size_t)J.cur * TCAP;
  float* tail_next = J.state + (size_t)(J.cur ^ 1) * TCAP;
  float* pend_g = J.state + PENDING_OFF;
  long long* pprev_g = reinterpret_cast<long long*>(J.state + PPREV_OFF);
  for (int n = tid; n < N; n += THREADS) hann[n] = (float)(0.5 - 0.5 * cospi(2.0 * n / N));
  for (int n = tid; n < H; n += THREADS) pend[n] = pend_g[n];
  long long p_prev = *pprev_g;
  __syncthreads();
  for (long long k = J.K0; k < J.K1; ++k) {
    long long p = 0, lo = 0;
    if (k > 0) {
      const long long a = (k * H * J.q) >> 10;
      lo = a - D > 0 ? a - D : 0;
      const int cnt = (int)(a + D - lo + 1);
      for (int i = tid; i < cnt + N - 1; i += THREADS) win[i] = xt(J, tail, lo + i);
      for (int i = tid; i < N; i += THREADS) tgt[i] = xt(J, tail, p_prev + H + i);
      __syncthreads();
      Best b{-INFINITY, 0x7fffffff, 0x7fffffff};
      if (tid < cnt) {
        float s = 0.f, e = 0.f;
#pragma unroll 8
        for (int n = 0; n < N; ++n) {
          const float x = win[tid + n];
          s = fmaf(tgt[n], x, s);
          e = fmaf(x, x, e);
        }
        const long long d = lo + tid - a;
        b = Best{s / sqrtf(EPS + e), (int)(d < 0 ? -d : d), tid};
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        Best r{__shfl_down_sync(0xffffffffu, b.s, o), __shfl_down_sync(0xffffffffu, b.d, o),
               __shfl_down_sync(0xffffffffu, b.c, o)};
        if (better(r, b)) b = r;
      }
      if ((tid & 31) == 0) part[tid >> 5] = b;
      __syncthreads();
      if (tid == 0) {
        Best r = part[0];
        for (int w = 1; w < THREADS / 32; ++w)
          if (better(part[w], r)) r = part[w];
        best_p = lo + r.c;
      }
      __syncthreads();
      p = best_p;
    }
    // overlap-add: y~[kH + n] = pending (frame k-1) + w[n] x~[p + n]; y~[kH, kH + H) is y[(k-1)H, kH)
    for (int n = tid; n < H; n += THREADS) {
      const float v0 = k > 0 ? win[p - lo + n] : xt(J, tail, p + n);
      const float v1 = k > 0 ? win[p - lo + H + n] : xt(J, tail, p + H + n);
      const float y = pend[n] + hann[n] * v0;
      const long long m = (k - 1) * H + n;
      if (k > 0 && m < J.E1) J.out[m - J.E0] = y;
      pend[n] = hann[H + n] * v1;
    }
    if (tid == 0 && J.pk) J.pk[k - J.K0] = (int32_t)p;
    p_prev = p;
    __syncthreads();
  }
  if (J.flush) return;
  for (int n = tid; n < H; n += THREADS) pend_g[n] = pend[n];
  if (tid == 0) *pprev_g = p_prev;
  for (long long j = J.ts1 + tid; j < J.L1; j += THREADS) tail_next[j - J.ts1] = xt(J, tail, j + H);
}

int quantize(double speed) {
  if (!(speed >= 0.0 && speed <= 8.0)) return -1;
  return (int)llrint(speed * 1024.0);
}

}  // namespace

struct fq3_tempo {
  int dev = 0, q = 1024, cur = 0;
  int64_t total_in = 0, frames = 0, emitted = 0, ts = 0;
  bool flushed = false;
  float* state = nullptr;
};


extern "C" int fq3_tempo_create(int32_t device, double speed, fq3_tempo** out) {
  if (!out) return tfail(FQ3_ERR_INVALID, "null argument");
  const int q = quantize(speed);
  if (q < FQ3_TEMPO_Q_MIN || q > FQ3_TEMPO_Q_MAX)
    return tfail(FQ3_ERR_INVALID, "speed must be in [0.25, 4.0] (round(speed * 1024) in [256, 4096])");
  if (q == 1024) return tfail(FQ3_ERR_INVALID, "speed 1 is the identity: no tempo state exists for it");
  DevGuard g(device);
  fq3_tempo* t = new fq3_tempo();
  t->dev = device;
  t->q = q;
  if (cudaMalloc(&t->state, STATE_FLOATS * sizeof(float)) != cudaSuccess) {
    delete t;
    return tfail(FQ3_ERR_CUDA, "cudaMalloc of the tempo state failed");
  }
  *out = t;
  return 0;
}

// host counters only: frame 0 rewrites the pending overlap and reads no p_{k-1}, the zeros in front are not stored
extern "C" int fq3_tempo_reset(fq3_tempo* t) {
  if (!t) return tfail(FQ3_ERR_INVALID, "null argument");
  t->total_in = t->frames = t->emitted = t->ts = 0;
  t->cur = 0;
  t->flushed = false;
  return 0;
}

extern "C" void fq3_tempo_destroy(fq3_tempo* t) {
  if (!t) return;
  DevGuard g(t->dev);
  cudaFree(t->state);
  delete t;
}

extern "C" int64_t fq3_tempo_released(int32_t q, int64_t total_in, int64_t n, int32_t flush) {
  if (q < FQ3_TEMPO_Q_MIN || q > FQ3_TEMPO_Q_MAX || total_in < 0 || n < 0) return -1;
  const int64_t K0 = ready_frames(total_in, q), E0 = std::max<int64_t>(0, K0 - 1) * H, L1 = total_in + n;
  if (flush) return (L1 * 1024 + q / 2) / q - E0;
  return std::max<int64_t>(0, ready_frames(L1, q) - 1) * H - E0;
}

extern "C" int fq3_tempo_process(fq3_tempo* const* tempos, int32_t n_streams, const float* in_dev,
                                 const int64_t* in_lens, const int32_t* flush, float* out_dev, int64_t out_cap,
                                 int32_t* pk_dev, int64_t pk_cap, void* stream_) {
  if (!tempos || n_streams <= 0 || !in_lens || !flush) return tfail(FQ3_ERR_INVALID, "null argument");
  if (((uintptr_t)in_dev | (uintptr_t)out_dev | (uintptr_t)pk_dev) & 3)
    return tfail(FQ3_ERR_INVALID, "misaligned buffer (float32 / int32 need 4-byte alignment)");
  const int dev = tempos[0] ? tempos[0]->dev : 0;
  std::vector<Job> jobs(n_streams);
  int64_t in_off = 0, out_off = 0, pk_off = 0;
  for (int b = 0; b < n_streams; ++b) {
    fq3_tempo* t = tempos[b];
    if (!t) return tfail(FQ3_ERR_INVALID, "null tempo handle");
    if (t->dev != dev) return tfail(FQ3_ERR_INVALID, "tempo handles of different devices");
    for (int a = 0; a < b; ++a)
      if (tempos[a] == t) return tfail(FQ3_ERR_INVALID, "tempo listed twice");
    if (t->flushed) return tfail(FQ3_ERR_STATE, "tempo already flushed (reset it to start a new stream)");
    if (in_lens[b] < 0) return tfail(FQ3_ERR_INVALID, "negative input length");
    Job& J = jobs[b];
    J.state = t->state;
    J.in = in_dev + in_off;
    J.q = t->q;
    J.cur = t->cur;
    J.flush = flush[b] != 0;
    J.L0 = t->total_in;
    J.L1 = t->total_in + in_lens[b];
    J.ts0 = t->ts;
    J.K0 = t->frames;
    J.E0 = t->emitted;
    if (J.flush) {
      J.E1 = (J.L1 * 1024 + t->q / 2) / t->q;
      J.K1 = std::max<int64_t>(J.K0, (J.E1 + H - 1) / H + 1);
      J.ts1 = J.ts0;
    } else {
      J.K1 = ready_frames(J.L1, t->q);
      J.E1 = std::max<int64_t>(0, J.K1 - 1) * H;
      J.ts1 = std::min<int64_t>(J.L1, std::max<int64_t>(0, reach_lo(J.K1, t->q) - H));
      if (J.L1 - J.ts1 > TCAP) return tfail(FQ3_ERR_INVALID, "internal: tempo tail exceeds its capacity");
    }
    J.out = out_dev + out_off;
    J.pk = pk_dev ? pk_dev + pk_off : nullptr;
    in_off += in_lens[b];
    out_off += J.E1 - J.E0;
    pk_off += J.K1 - J.K0;
  }
  if (in_off > 0 && !in_dev) return tfail(FQ3_ERR_INVALID, "null input buffer");
  if (out_off > 0 && !out_dev) return tfail(FQ3_ERR_INVALID, "null output buffer");
  if (out_off > out_cap) return tfail(FQ3_ERR_INVALID, "output buffer smaller than the released samples");
  if (pk_dev && pk_off > pk_cap) return tfail(FQ3_ERR_INVALID, "position buffer smaller than the frames run");
  DevGuard g(dev);
  cudaStream_t stream = (cudaStream_t)stream_;
  Job* d_jobs = nullptr;
  cudaError_t e = cudaMallocAsync(&d_jobs, sizeof(Job) * n_streams, stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d_jobs, jobs.data(), sizeof(Job) * n_streams, cudaMemcpyHostToDevice, stream);
  if (e == cudaSuccess) {
    tempo_kernel<<<n_streams, THREADS, 0, stream>>>(d_jobs);
    e = cudaGetLastError();
  }
  if (d_jobs) cudaFreeAsync(d_jobs, stream);
  if (e != cudaSuccess) return tfail(FQ3_ERR_CUDA, cudaGetErrorString(e));
  for (int b = 0; b < n_streams; ++b) {
    fq3_tempo* t = tempos[b];
    const Job& J = jobs[b];
    t->total_in = J.L1;
    t->frames = J.K1;
    t->emitted = J.E1;
    t->ts = J.ts1;
    t->cur ^= 1;
    t->flushed = J.flush;
  }
  return 0;
}

extern "C" const char* fq3_tempo_last_error(void) { return g_terr; }
