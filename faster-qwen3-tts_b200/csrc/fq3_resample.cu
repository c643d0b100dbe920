// fq3_resample.cu -- output sample rate, pitch, gain and encoding: a rational polyphase resampler of 24 kHz PCM that is
// already on the device, with the gain and the encoding (f32, s16, G.711 mu-law / A-law) applied in the store, for any
// number of streams in one launch.  The algorithm is fixed exactly (DESIGN.md, "Output rate and encoding" and "Pitch and
// gain"; faster_qwen3_tts/resample.py restates the counts; oracle/resample_oracle.py restates the arithmetic in float64
// at rho 256, tests/pitch_oracle.py at every rho):
//
//   R in {8000, 16000, 22050, 24000, 32000, 44100, 48000}; rho in [128, 512] (the pitch ratio is rho / 256; 256 is no
//   pitch shift).  (L, M) = (256 R, 24000 rho) reduced by their gcd, m = max(L, M), half = 32 m.
//   h = firwin(2 half + 1, 0.9 / m, Kaiser beta 8.6), scaled to unit DC gain, designed here in double.
//   y[n] = g * (L * sum_j h[j] x[(n M + half - j) / L]) over the j with (n M + half - j) a non-negative multiple of L
//   and the index in [0, N); x is zero outside [0, N); g is the stream's float32 gain, one fp32 multiply (g = 1 leaves
//   the sum's bits).  A flushed stream of N samples has ceil(N L / M) outputs.
//   L == M (R = 24000 at rho 256, 48000 at rho 512) is the encode-only case: h = {1}, half = 0.  R = 24000 at rho 256
//   with f32 and g = 1 is the identity: callers pass the PCM through (fq3_resample_create refuses it).
//
// Output n is released once input floor((n M + half) / L) exists, so the counts of a push are a function of the stream's
// totals alone: the host sizes every buffer before the launch and nothing is read back.  Output n is a dot product over
// fixed input indices in a fixed order (phase p = (n M + half) mod L, taps k = 0 .. K_p - 1 with input top - k, top =
// floor((n M + half) / L)), so the bits do not depend on how the input was split into pushes, nor on which streams share
// the launch.
//
// Outputs are independent: the grid is one CTA per (stream, tile of TILE outputs), one thread per output.  A CTA stages
// the input span its tile reads in shared memory.  Where the whole phase table fits beside that span in 48 KB (every
// plain rate, up to 41 KB at 22.05 kHz, and the small pitched tables) the CTA stages the table too; otherwise (most
// pitched tables, up to 0.65 MB) each thread reads its output's phase row from the L2-resident table in global memory.
// The choice is a function of (L, M, half) alone, so host and kernel make it alike, and both paths sum the same fp32
// values in the same order: the bits do not depend on the path.  New samples are read in place from the caller's
// packed buffer; the per-stream device state is the last TC = ceil(2 half / L) input samples, in two alternating
// buffers, so the CTA that writes the next tail never overwrites the one the other CTAs of the same launch read.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include <algorithm>
#include <cstring>
#include <list>
#include <map>
#include <tuple>
#include <mutex>
#include <utility>
#include <vector>

#include "../../include/fq3_engine.h"

namespace {

constexpr int TILE = 256;               // outputs per CTA, one per thread
constexpr int TCAP = 384;               // tail buffer capacity: the largest tail is 384 samples (8 kHz, rho 512)
constexpr int SMEM_MAX = 48 * 1024;     // no opt-in needed: a table is staged only where it fits beside its span

thread_local char g_rerr[256] = "";
int rfail(int code, const char* msg) {
  snprintf(g_rerr, sizeof(g_rerr), "%s", msg);
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

int64_t gcd64(int64_t a, int64_t b) {
  while (b) {
    const int64_t t = a % b;
    a = b;
    b = t;
  }
  return a;
}

bool valid_rate(int rate) {
  switch (rate) {
    case 8000: case 16000: case 22050: case 24000: case 32000: case 44100: case 48000: return true;
    default: return false;
  }
}

int sample_bytes(int enc) { return enc == FQ3_ENC_F32 ? 4 : enc == FQ3_ENC_S16 ? 2 : 1; }

// floats of input a tile of TILE outputs reads, at most
__host__ __device__ inline long long span_floats(int L, int M, int half) {
  return ((TILE - 1) * (long long)M + 2 * half) / L + 2;
}

// whether a CTA stages the L x kmax phase table in shared memory (beside its input span) or reads rows from global
__host__ __device__ inline bool stages_table(int L, int M, int half, int kmax) {
  return ((long long)L * kmax + span_floats(L, M, half)) * (long long)sizeof(float) <= (long long)SMEM_MAX;
}

struct Ratio {
  int L, M, half;
  int kmax() const { return 2 * half / L + 1; }        // taps of phase 0, the most of any phase
  int tail() const { return (2 * half + L - 1) / L; }  // ceil(2 half / L)
};

bool valid_pitch(int rho) { return rho >= FQ3_RESAMPLE_PITCH_MIN && rho <= FQ3_RESAMPLE_PITCH_MAX; }

// (L, M) = (256 R, 24000 rho) / gcd; L == M is the encode-only identity filter: one tap, no look-ahead.  At rho 256
// this is (R, 24000) / gcd, with 24000 the encode-only rate.
Ratio ratio_of(int rate, int rho) {
  const int64_t a = (int64_t)rate * FQ3_RESAMPLE_PITCH_ONE, b = (int64_t)FQ3_RESAMPLE_IN_RATE * rho;
  const int64_t g = gcd64(a, b);
  const int L = (int)(a / g), M = (int)(b / g);
  if (L == M) return Ratio{1, 1, 0};
  return Ratio{L, M, FQ3_RESAMPLE_HALF_PER_M * (L > M ? L : M)};
}

// modified Bessel function of the first kind, order 0: the power series, to double precision for x <= 2 beta
double bessel_i0(double x) {
  double sum = 1.0, term = 1.0;
  const double q = 0.25 * x * x;
  for (int k = 1; k < 200; ++k) {
    term *= q / ((double)k * k);
    sum += term;
    if (term < 1e-18 * sum) break;
  }
  return sum;
}

// firwin(2 half + 1, 0.9 / m, window=("kaiser", 8.6)), scaled to unit DC gain
std::vector<double> design(int rate, int rho) {
  const Ratio r = ratio_of(rate, rho);
  if (r.half == 0) return {1.0};
  const int n = 2 * r.half + 1;
  const double m = r.L > r.M ? r.L : r.M;
  const double fc = FQ3_RESAMPLE_CUTOFF / m, i0b = bessel_i0(FQ3_RESAMPLE_BETA);
  std::vector<double> h(n);
  double s = 0.0;
  for (int i = 0; i < n; ++i) {
    const double t = i - r.half;
    const double a = M_PI * fc * t;
    const double sinc = t == 0 ? 1.0 : sin(a) / a;
    const double u = t / r.half;
    const double w = bessel_i0(FQ3_RESAMPLE_BETA * sqrt(1.0 - u * u)) / i0b;
    h[i] = fc * sinc * w;
    s += h[i];
  }
  for (double& v : h) v /= s;
  return h;
}

// one device phase table per (device, rate, rho), shared by every stream at that rate and pitch: row p holds
// L * h[p + L k] for k < K_p, zero-padded to kmax.  Plain tables (rho 256, seven at most) are kept for the process's
// lifetime.  Pitched tables are counted by the handles that use them; once unreferenced they stay cached, and beyond
// FQ3_RESAMPLE_TABLE_CACHE unreferenced ones the least recently released is freed.
struct Table {
  float* d = nullptr;
  int64_t bytes = 0;
  int refs = 0;
};
using TabKey = std::tuple<int, int, int>;   // (device, rate, rho)
std::mutex g_tab_mu;
std::map<TabKey, Table> g_tabs;
std::list<TabKey> g_idle;                   // unreferenced pitched tables, least recently released first

int table_for(int dev, int rate, int rho, float** out) {
  std::lock_guard<std::mutex> lk(g_tab_mu);
  const TabKey key{dev, rate, rho};
  auto it = g_tabs.find(key);
  if (it == g_tabs.end()) {
    const Ratio r = ratio_of(rate, rho);
    const std::vector<double> h = design(rate, rho);
    const int kmax = r.kmax();
    std::vector<float> tab((size_t)r.L * kmax, 0.f);
    for (int p = 0; p < r.L; ++p)
      for (int k = 0; p + r.L * k <= 2 * r.half; ++k) tab[(size_t)p * kmax + k] = (float)(r.L * h[p + r.L * k]);
    float* d = nullptr;
    if (cudaMalloc(&d, tab.size() * sizeof(float)) != cudaSuccess)
      return rfail(FQ3_ERR_CUDA, "cudaMalloc of a phase table failed");
    if (cudaMemcpy(d, tab.data(), tab.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) {
      cudaFree(d);
      return rfail(FQ3_ERR_CUDA, "upload of a phase table failed");
    }
    it = g_tabs.emplace(key, Table{d, (int64_t)(tab.size() * sizeof(float)), 0}).first;
  }
  if (rho != FQ3_RESAMPLE_PITCH_ONE && it->second.refs++ == 0) g_idle.remove(key);
  *out = it->second.d;
  return 0;
}

// a handle of a pitched table is gone: an unreferenced table joins the idle list, whose oldest entries beyond
// FQ3_RESAMPLE_TABLE_CACHE are freed
void table_release(int dev, int rate, int rho) {
  if (rho == FQ3_RESAMPLE_PITCH_ONE) return;
  std::lock_guard<std::mutex> lk(g_tab_mu);
  const TabKey key{dev, rate, rho};
  auto it = g_tabs.find(key);
  if (it == g_tabs.end() || --it->second.refs > 0) return;
  g_idle.push_back(key);
  while ((int)g_idle.size() > FQ3_RESAMPLE_TABLE_CACHE) {
    const TabKey old = g_idle.front();
    g_idle.pop_front();
    auto o = g_tabs.find(old);
    {
      DevGuard g(std::get<0>(old));
      cudaFree(o->second.d);
    }
    g_tabs.erase(o);
  }
}

int64_t ceil_div(int64_t a, int64_t b) { return a >= 0 ? (a + b - 1) / b : -((-a) / b); }

// outputs released once total_in samples exist (and are flushed, when final)
int64_t emitted(const Ratio& r, int64_t total_in, bool final) {
  const int64_t all = ceil_div(total_in * r.L, r.M);
  if (final) return all;
  const int64_t ready = ceil_div(total_in * r.L - r.half, r.M);
  return std::min<int64_t>(all, std::max<int64_t>(0, ready));
}

struct Job {
  const float* tail;       // x[L0 - tc, L0) (entries of negative index are never read)
  float* tail_next;        // <- x[L1 - tc, L1), written by the job's first tile unless the stream flushes
  const float* in;         // new samples x[L0, L1)
  const float* tab;        // L x kmax phase table
  unsigned char* out;      // encoded g * y[E0, E1)
  long long L0, L1, E0, E1;
  int L, M, half, kmax, tc, enc, write_tail;
  float gain;
};

struct Tile {
  int job, n0;             // outputs [E0 + n0, E0 + min(n0 + TILE, E1 - E0))
};

__device__ __forceinline__ float xin(const Job& J, long long i) {
  if (i < 0 || i >= J.L1) return 0.f;
  if (i < J.L0) return J.tail[i - (J.L0 - J.tc)];
  return J.in[i - J.L0];
}

// serving.to_pcm16: clip(x * 32768, -32768, 32767), then truncation toward zero, in fp32
__device__ __forceinline__ int to_s16(float x) { return (int)fminf(fmaxf(x * 32768.f, -32768.f), 32767.f); }

// ITU-T G.711 mu-law of a 16-bit sample, as audioop.lin2ulaw: the 14-bit magnitude, clipped, biased and segmented
__device__ __forceinline__ unsigned char to_ulaw(int s) {
  int v = s >> 2, mask = 0xFF;
  if (v < 0) {
    v = -v;
    mask = 0x7F;
  }
  if (v > 8159) v = 8159;
  v += 0x84 >> 2;
  int seg = 0;
  while (seg < 8 && v > (0x40 << seg) - 1) ++seg;   // seg_uend = 0x3F, 0x7F, ..., 0x1FFF
  if (seg >= 8) return (unsigned char)(0x7F ^ mask);
  return (unsigned char)(((seg << 4) | ((v >> (seg + 1)) & 0xF)) ^ mask);
}

// ITU-T G.711 A-law of a 16-bit sample, as audioop.lin2alaw: the 13-bit magnitude, segmented, even bits inverted
__device__ __forceinline__ unsigned char to_alaw(int s) {
  int v = s >> 3, mask = 0xD5;
  if (v < 0) {
    v = -v - 1;
    mask = 0x55;
  }
  int seg = 0;
  while (seg < 8 && v > (0x20 << seg) - 1) ++seg;   // seg_aend = 0x1F, 0x3F, ..., 0xFFF
  if (seg >= 8) return (unsigned char)(0x7F ^ mask);
  const int q = seg < 2 ? (v >> 1) & 0xF : (v >> seg) & 0xF;
  return (unsigned char)(((seg << 4) | q) ^ mask);
}

__global__ void __launch_bounds__(TILE) resample_kernel(const Job* __restrict__ jobs, const Tile* __restrict__ tiles) {
  extern __shared__ float smem[];
  const Tile T = tiles[blockIdx.x];
  const Job J = jobs[T.job];
  const int tid = threadIdx.x;
  const long long n0 = J.E0 + T.n0;
  const int cnt = (int)min((long long)TILE, J.E1 - n0);
  if (J.write_tail && T.n0 == 0)
    for (int j = tid; j < J.tc; j += TILE) J.tail_next[j] = xin(J, J.L1 - J.tc + j);
  if (cnt <= 0) return;
  const bool staged = stages_table(J.L, J.M, J.half, J.kmax);
  float* xs = smem + (staged ? J.L * J.kmax : 0);
  const long long top0 = (n0 * J.M + J.half) / J.L;
  const long long lo = top0 - (J.kmax - 1);
  const int span = (int)(((n0 + cnt - 1) * J.M + J.half) / J.L - lo + 1);
  if (staged)
    for (int i = tid; i < J.L * J.kmax; i += TILE) smem[i] = J.tab[i];
  for (int i = tid; i < span; i += TILE) xs[i] = xin(J, lo + i);
  __syncthreads();
  if (tid >= cnt) return;
  const long long n = n0 + tid;
  const long long t = n * J.M + J.half;
  const int p = (int)(t % J.L);
  const int K = (2 * J.half - p) / J.L + 1;
  const float* x = xs + (t / J.L - lo);
  float acc = 0.f;
  if (staged) {
    const float* g = smem + p * J.kmax;
    for (int k = 0; k < K; ++k) acc = fmaf(g[k], x[-k], acc);
  } else {
    const float* __restrict__ g = J.tab + (size_t)p * J.kmax;
#pragma unroll 4
    for (int k = 0; k < K; ++k) acc = fmaf(__ldg(g + k), x[-k], acc);
  }
  acc *= J.gain;
  const long long o = n - J.E0;
  switch (J.enc) {
    case FQ3_ENC_F32: reinterpret_cast<float*>(J.out)[o] = acc; break;
    case FQ3_ENC_S16: reinterpret_cast<int16_t*>(J.out)[o] = (int16_t)to_s16(acc); break;
    case FQ3_ENC_ULAW: J.out[o] = to_ulaw(to_s16(acc)); break;
    default: J.out[o] = to_alaw(to_s16(acc)); break;
  }
}

}  // namespace

struct fq3_resample {
  int dev = 0, rate = 0, rho = FQ3_RESAMPLE_PITCH_ONE, enc = 0, cur = 0;
  Ratio r{1, 1, 0};
  float gain = 1.f;
  int64_t total_in = 0, emitted = 0;
  bool flushed = false;
  float* state = nullptr;   // two TCAP tail buffers
  const float* tab = nullptr;
};

extern "C" int fq3_resample_create_pitch(int32_t device, int32_t out_rate, int32_t pitch_rho, int32_t encoding,
                                         fq3_resample** out) {
  if (!out) return rfail(FQ3_ERR_INVALID, "null argument");
  if (!valid_rate(out_rate))
    return rfail(FQ3_ERR_INVALID, "output rate must be one of 8000, 16000, 22050, 24000, 32000, 44100, 48000");
  if (!valid_pitch(pitch_rho)) return rfail(FQ3_ERR_INVALID, "pitch rho must be in [128, 512]");
  if (encoding < FQ3_ENC_F32 || encoding > FQ3_ENC_ALAW) return rfail(FQ3_ERR_INVALID, "unknown encoding");
  DevGuard g(device);
  float* tab = nullptr;
  if (int rc = table_for(device, out_rate, pitch_rho, &tab)) return rc;
  fq3_resample* s = new fq3_resample();
  s->dev = device;
  s->rate = out_rate;
  s->rho = pitch_rho;
  s->enc = encoding;
  s->r = ratio_of(out_rate, pitch_rho);
  s->tab = tab;
  if (cudaMalloc(&s->state, 2 * TCAP * sizeof(float)) != cudaSuccess) {
    table_release(device, out_rate, pitch_rho);
    delete s;
    return rfail(FQ3_ERR_CUDA, "cudaMalloc of the resampler state failed");
  }
  *out = s;
  return 0;
}

extern "C" int fq3_resample_create(int32_t device, int32_t out_rate, int32_t encoding, fq3_resample** out) {
  if (out_rate == FQ3_RESAMPLE_IN_RATE && encoding == FQ3_ENC_F32)
    return rfail(FQ3_ERR_INVALID, "24000 Hz f32 is the identity: no resampler state exists for it");
  return fq3_resample_create_pitch(device, out_rate, FQ3_RESAMPLE_PITCH_ONE, encoding, out);
}

extern "C" int fq3_resample_set_gain(fq3_resample* s, float gain) {
  if (!s) return rfail(FQ3_ERR_INVALID, "null argument");
  if (!(gain >= 0.f && gain <= 1e6f)) return rfail(FQ3_ERR_INVALID, "gain must be a finite non-negative number");
  s->gain = gain;
  return 0;
}

// host counters only: reads below input index 0 are zeros and never touch the stored tail
extern "C" int fq3_resample_reset(fq3_resample* s) {
  if (!s) return rfail(FQ3_ERR_INVALID, "null argument");
  s->total_in = s->emitted = 0;
  s->cur = 0;
  s->flushed = false;
  return 0;
}

extern "C" void fq3_resample_destroy(fq3_resample* s) {
  if (!s) return;
  DevGuard g(s->dev);
  cudaFree(s->state);
  table_release(s->dev, s->rate, s->rho);
  delete s;
}

extern "C" int64_t fq3_resample_released_pitch(int32_t out_rate, int32_t pitch_rho, int64_t total_in, int64_t n,
                                               int32_t flush) {
  if (!valid_rate(out_rate) || !valid_pitch(pitch_rho) || total_in < 0 || n < 0) return -1;
  const Ratio r = ratio_of(out_rate, pitch_rho);
  return emitted(r, total_in + n, flush != 0) - emitted(r, total_in, false);
}

extern "C" int64_t fq3_resample_released(int32_t out_rate, int64_t total_in, int64_t n, int32_t flush) {
  return fq3_resample_released_pitch(out_rate, FQ3_RESAMPLE_PITCH_ONE, total_in, n, flush);
}

extern "C" int32_t fq3_resample_taps_pitch(int32_t out_rate, int32_t pitch_rho, double* out, int32_t cap) {
  if (!valid_rate(out_rate) || !valid_pitch(pitch_rho)) return -1;
  const std::vector<double> h = design(out_rate, pitch_rho);
  if (out)
    for (int i = 0; i < (int)h.size() && i < cap; ++i) out[i] = h[i];
  return (int32_t)h.size();
}

extern "C" int32_t fq3_resample_taps(int32_t out_rate, double* out, int32_t cap) {
  return fq3_resample_taps_pitch(out_rate, FQ3_RESAMPLE_PITCH_ONE, out, cap);
}

extern "C" int64_t fq3_resample_table_bytes(int32_t device) {
  std::lock_guard<std::mutex> lk(g_tab_mu);
  int64_t total = 0;
  for (const auto& kv : g_tabs)
    if (std::get<0>(kv.first) == device) total += kv.second.bytes;
  return total;
}

extern "C" int fq3_resample_process(fq3_resample* const* rs, int32_t n_streams, const float* in_dev,
                                    const int64_t* in_lens, const int32_t* flush, void* out_dev, int64_t out_cap,
                                    void* stream_) {
  if (!rs || n_streams <= 0 || !in_lens || !flush) return rfail(FQ3_ERR_INVALID, "null argument");
  if ((uintptr_t)in_dev & 3) return rfail(FQ3_ERR_INVALID, "misaligned input buffer (float32 needs 4-byte alignment)");
  if ((uintptr_t)out_dev & (FQ3_RESAMPLE_ALIGN - 1))
    return rfail(FQ3_ERR_INVALID, "misaligned output buffer (each stream's slice starts 16-byte aligned)");
  const int dev = rs[0] ? rs[0]->dev : 0;
  std::vector<Job> jobs(n_streams);
  std::vector<Tile> tiles;
  int64_t in_off = 0, out_off = 0;
  size_t smem = 0;
  for (int b = 0; b < n_streams; ++b) {
    fq3_resample* s = rs[b];
    if (!s) return rfail(FQ3_ERR_INVALID, "null resampler handle");
    if (s->dev != dev) return rfail(FQ3_ERR_INVALID, "resampler handles of different devices");
    for (int a = 0; a < b; ++a)
      if (rs[a] == s) return rfail(FQ3_ERR_INVALID, "resampler listed twice");
    if (s->flushed) return rfail(FQ3_ERR_STATE, "resampler already flushed (reset it to start a new stream)");
    if (in_lens[b] < 0) return rfail(FQ3_ERR_INVALID, "negative input length");
    const Ratio& r = s->r;
    Job& J = jobs[b];
    J.L = r.L;
    J.M = r.M;
    J.half = r.half;
    J.kmax = r.kmax();
    J.tc = r.tail();
    J.enc = s->enc;
    J.gain = s->gain;
    J.tab = s->tab;
    J.tail = s->state + (size_t)s->cur * TCAP;
    J.tail_next = s->state + (size_t)(s->cur ^ 1) * TCAP;
    J.in = in_dev + in_off;
    J.L0 = s->total_in;
    J.L1 = s->total_in + in_lens[b];
    J.E0 = s->emitted;
    J.E1 = emitted(r, J.L1, flush[b] != 0);
    J.write_tail = flush[b] == 0 && in_lens[b] > 0 && J.tc > 0;
    if (J.tc > TCAP) return rfail(FQ3_ERR_INVALID, "internal: resampler tail exceeds its capacity");
    out_off = (out_off + FQ3_RESAMPLE_ALIGN - 1) / FQ3_RESAMPLE_ALIGN * FQ3_RESAMPLE_ALIGN;
    J.out = (unsigned char*)out_dev + out_off;
    out_off += (J.E1 - J.E0) * sample_bytes(s->enc);
    in_off += in_lens[b];
    const int64_t n_out = J.E1 - J.E0;
    for (int64_t n0 = 0; n0 < n_out; n0 += TILE) tiles.push_back(Tile{b, (int)n0});
    if (n_out == 0 && J.write_tail) tiles.push_back(Tile{b, 0});
    if (n_out > 0) {
      const size_t tab = stages_table(r.L, r.M, r.half, J.kmax) ? (size_t)r.L * J.kmax : 0;
      smem = std::max(smem, (tab + (size_t)span_floats(r.L, r.M, r.half)) * sizeof(float));
    }
  }
  if (in_off > 0 && !in_dev) return rfail(FQ3_ERR_INVALID, "null input buffer");
  if (out_off > 0 && !out_dev) return rfail(FQ3_ERR_INVALID, "null output buffer");
  if (out_off > out_cap) return rfail(FQ3_ERR_INVALID, "output buffer smaller than the released samples");
  if (smem > (size_t)SMEM_MAX) return rfail(FQ3_ERR_INVALID, "internal: resampler tile exceeds shared memory");
  if (!tiles.empty()) {
    DevGuard g(dev);
    cudaStream_t stream = (cudaStream_t)stream_;
    // jobs, then tiles, in one stream-ordered allocation
    const size_t jb = sizeof(Job) * n_streams, tb = sizeof(Tile) * tiles.size();
    std::vector<unsigned char> blob(jb + tb);
    memcpy(blob.data(), jobs.data(), jb);
    memcpy(blob.data() + jb, tiles.data(), tb);
    void* d = nullptr;
    cudaError_t e = cudaMallocAsync(&d, blob.size(), stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d, blob.data(), blob.size(), cudaMemcpyHostToDevice, stream);
    if (e == cudaSuccess) {
      resample_kernel<<<(unsigned)tiles.size(), TILE, smem, stream>>>(
          (const Job*)d, (const Tile*)((unsigned char*)d + jb));
      e = cudaGetLastError();
    }
    if (d) cudaFreeAsync(d, stream);
    if (e != cudaSuccess) return rfail(FQ3_ERR_CUDA, cudaGetErrorString(e));
  }
  for (int b = 0; b < n_streams; ++b) {
    fq3_resample* s = rs[b];
    const Job& J = jobs[b];
    s->total_in = J.L1;
    s->emitted = J.E1;
    if (J.write_tail) s->cur ^= 1;
    s->flushed = flush[b] != 0;
  }
  return 0;
}

extern "C" const char* fq3_resample_last_error(void) { return g_rerr; }
