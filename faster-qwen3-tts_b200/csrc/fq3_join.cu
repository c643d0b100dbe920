// fq3_join.cu -- the join of a segmented request (DESIGN.md, "Long inputs"; faster_qwen3_tts/join.py restates the rule,
// tests/join_oracle.py the arithmetic): the 24 kHz float32 PCM of its S segments, which are decoded as separate rows and
// finish in any order, becomes one stream, in segment order:
//
//   out = P_0 zeros · seg_0 · P_1 zeros · seg_1 · ... · P_{S-1} zeros · seg_{S-1} · P_S zeros,   P_k = 24 * pauses_ms[k]
//
// fq3_join_create(pause_ms) is the plan [0, P, ..., P, 0].  The leading P_0 zeros are released with segment 0's first
// push, the trailing P_S zeros in the call that completes the stream.
//
// with a raised-cosine fade at every inner boundary: sample n of segment k (length L) is x * a * b in fp32, in that
// order, with a = w[n] for k > 0 and n < F (else 1) and b = w[L - 1 - n] for k < S - 1 and L - 1 - n < F (else 1), where
// F = FQ3_JOIN_FADE (5 ms) and w[i] = float32(0.5 - 0.5 cos(pi (i + 0.5) / F)) (double on the host).
//
// Release.  The segment being played (`cur`) streams out as its samples arrive, except its last F samples while it has
// not ended (their fade-out depends on where it ends), which wait in a ping-pong tail of F floats.  Samples of a later
// segment stay on the device, in one buffer per push, until every earlier segment has ended; then they are released in
// the same call.  So the samples a call releases are a function of the lengths and end flags alone: the host sizes every
// buffer before the launch (fq3_join_released) and no value ever comes back.  The output does not depend on how the
// segments were split into pushes.
//
// One launch per call covers every join in it: the host cuts the call into pieces (copy with fade, copy, zeros), each at
// most PIECE samples, one CTA per piece.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include <algorithm>
#include <map>
#include <vector>

#include "../../include/fq3_engine.h"

namespace {

constexpr int F = FQ3_JOIN_FADE;
constexpr int THREADS = 256;
constexpr int64_t PIECE = 8192;

thread_local char g_jerr[256] = "";
int jfail(int code, const char* msg) {
  snprintf(g_jerr, sizeof(g_jerr), "%s", msg);
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

struct Fade {
  float w[F];
};

Fade make_fade() {
  Fade f;
  for (int i = 0; i < F; ++i) f.w[i] = (float)(0.5 - 0.5 * cos(M_PI * (i + 0.5) / F));
  return f;
}

// dst[i] = src[i] * a * b (fades of segment position pos + i, segment length L; L < 0 while it has not ended), or 0
// when src is null
struct Piece {
  const float* src;
  float* dst;
  long long n, pos, L;
  int fin, fout;
};

__global__ void __launch_bounds__(THREADS) join_kernel(const Piece* __restrict__ pieces, Fade fade) {
  const Piece P = pieces[blockIdx.x];
  for (long long i = threadIdx.x; i < P.n; i += THREADS) {
    if (!P.src) {
      P.dst[i] = 0.f;
      continue;
    }
    float y = P.src[i];
    const long long p = P.pos + i;
    if (P.fin && p < F) y = y * fade.w[p];
    if (P.fout && P.L >= 0 && P.L - 1 - p < F) y = y * fade.w[P.L - 1 - p];
    P.dst[i] = y;
  }
}

struct Chunk {
  float* p;
  int64_t pos, n;   // segment positions [pos, pos + n)
};

struct Seg {
  int64_t total = 0;
  bool ended = false;
  std::vector<Chunk> chunks;   // held samples of a segment after `cur`
};

}  // namespace

struct fq3_join {
  int dev = 0, S = 0, cur = 0, pp = 0;
  bool lead_done = false, tail_done = false;   // the leading / trailing zeros have been released
  std::vector<int64_t> pause;                  // S + 1 zero runs, in samples: before segment 0, between, after the last
  int64_t out_pos = 0, released = 0;   // of segment cur: samples [out_pos, segs[cur].total) are in tail[pp]
  float* tail = nullptr;               // 2 x F
  std::vector<Seg> segs;
};

namespace {

void free_chunks(fq3_join* j) {
  for (Seg& s : j->segs)
    for (Chunk& c : s.chunks) cudaFree(c.p);
}

struct Push {
  int64_t in_off, n;
  bool end;
};

// One join's share of a call.  `pushes`: segment -> its push.  Without `run` only counts (and validates); with it
// appends the pieces, writes released samples from out, allocates the held chunks and updates the state.
int plan(fq3_join* j, const std::map<int, Push>& pushes, bool run, const float* in_dev, float* out, int64_t* n_out,
         std::vector<Piece>* pieces, std::vector<float*>* to_free, cudaStream_t stream) {
  for (auto& kv : pushes) {
    if (kv.first < 0 || kv.first >= j->S) return jfail(FQ3_ERR_INVALID, "segment index out of range");
    if (j->segs[kv.first].ended) return jfail(FQ3_ERR_STATE, "push to a segment that has ended");
    if (kv.second.n < 0) return jfail(FQ3_ERR_INVALID, "negative input length");
  }
  int64_t emitted = 0;
  const bool lead = !j->lead_done && pushes.count(0);
  float* tail_old = j->tail + (size_t)j->pp * F;
  float* tail_new = j->tail + (size_t)(j->pp ^ 1) * F;
  auto add = [&](const float* src, float* dst, int64_t n, int64_t pos, int64_t L, bool fin, bool fout) {
    for (int64_t o = 0; o < n; o += PIECE)
      pieces->push_back(Piece{src ? src + o : nullptr, dst + o, std::min(PIECE, n - o), pos + o, L, fin, fout});
  };
  // copy segment positions [a, b) of segment k to dst from wherever they are: tail (k == j->cur at entry), chunks, or
  // this call's input
  auto gather = [&](int k, bool was_cur, int64_t a, int64_t b, float* dst, bool fade, int64_t L) {
    const Seg& s = j->segs[k];
    auto it = pushes.find(k);
    const int64_t in0 = s.total;   // input covers [in0, in0 + n)
    const bool fin = fade && k > 0, fout = fade && k < j->S - 1;
    auto span = [&](const float* base, int64_t lo, int64_t hi) {   // base holds segment position lo at base[0]
      const int64_t x = std::max(a, lo), y = std::min(b, hi);
      if (x < y) add(base + (x - lo), dst + (x - a), y - x, x, L, fin, fout);
    };
    if (was_cur) span(tail_old, j->out_pos, in0);
    else
      for (const Chunk& c : s.chunks) span(c.p, c.pos, c.pos + c.n);
    if (it != pushes.end()) span(in_dev + it->second.in_off, in0, in0 + it->second.n);
  };
  if (lead) {   // the leading zeros, with segment 0's first push
    if (run) add(nullptr, out, j->pause[0], 0, -1, false, false);
    emitted += j->pause[0];
  }
  // the state after this call, applied only when `run`
  int cur = j->cur;
  int64_t out_pos = j->out_pos;
  bool tail = false;
  for (int k = cur;; ++k) {
    const Seg& s = j->segs[k];
    auto it = pushes.find(k);
    const int64_t total = s.total + (it != pushes.end() ? it->second.n : 0);
    const bool ended = s.ended || (it != pushes.end() && it->second.end);
    const bool was_cur = k == j->cur;
    const int64_t from = was_cur ? j->out_pos : 0;
    const int64_t upto = (ended || k == j->S - 1) ? total : std::max(from, total - F);
    if (run) {
      gather(k, was_cur, from, upto, out + emitted, true, ended ? total : -1);
      if (!ended && upto < total) gather(k, was_cur, upto, total, tail_new, false, -1);
      if (!was_cur)
        for (const Chunk& c : s.chunks) to_free->push_back(c.p);
    }
    emitted += upto - from;
    cur = k;
    out_pos = upto;
    const int64_t P = j->pause[k + 1];   // the zeros after segment k
    if (k == j->S - 1) {
      tail = ended && !j->tail_done;
      if (tail) {
        if (run) add(nullptr, out + emitted, P, 0, -1, false, false);
        emitted += P;
      }
      break;
    }
    if (!ended) break;
    if (run) add(nullptr, out + emitted, P, 0, -1, false, false);
    emitted += P;
  }
  if (n_out) *n_out = emitted;
  if (!run) return 0;
  // later segments keep their new samples on the device
  for (auto& kv : pushes) {
    const int k = kv.first;
    const Push& p = kv.second;
    if (k > cur && p.n > 0) {
      float* buf = nullptr;
      if (cudaMallocAsync(&buf, sizeof(float) * p.n, stream) != cudaSuccess)
        return jfail(FQ3_ERR_CUDA, "cudaMallocAsync of a held segment buffer failed");
      add(in_dev + p.in_off, buf, p.n, 0, -1, false, false);
      j->segs[k].chunks.push_back(Chunk{buf, j->segs[k].total, p.n});
    }
  }
  for (int k = j->cur; k < cur; ++k) j->segs[k].chunks.clear();
  if (cur != j->cur) j->segs[cur].chunks.clear();
  for (auto& kv : pushes) {
    j->segs[kv.first].total += kv.second.n;
    j->segs[kv.first].ended = j->segs[kv.first].ended || kv.second.end;
  }
  j->cur = cur;
  j->out_pos = out_pos;
  j->lead_done = j->lead_done || lead;
  j->tail_done = j->tail_done || tail;
  j->pp ^= 1;
  j->released += emitted;
  return 0;
}

// the pushes of a call, grouped per join
int group(fq3_join* const* joins, int32_t n_joins, int32_t n_pushes, const int32_t* join_of, const int32_t* seg,
          const int64_t* lens, const int32_t* ends, std::vector<std::map<int, Push>>* per) {
  if (!joins || n_joins <= 0 || n_pushes < 0 || (n_pushes && (!join_of || !seg || !lens || !ends)))
    return jfail(FQ3_ERR_INVALID, "null argument");
  for (int b = 0; b < n_joins; ++b) {
    if (!joins[b]) return jfail(FQ3_ERR_INVALID, "null join handle");
    if (joins[b]->dev != joins[0]->dev) return jfail(FQ3_ERR_INVALID, "join handles of different devices");
    for (int a = 0; a < b; ++a)
      if (joins[a] == joins[b]) return jfail(FQ3_ERR_INVALID, "join listed twice");
  }
  per->assign(n_joins, {});
  int64_t off = 0;
  for (int i = 0; i < n_pushes; ++i) {
    if (join_of[i] < 0 || join_of[i] >= n_joins) return jfail(FQ3_ERR_INVALID, "push of an unknown join");
    if (lens[i] < 0) return jfail(FQ3_ERR_INVALID, "negative input length");
    if (!(*per)[join_of[i]].emplace(seg[i], Push{off, lens[i], ends[i] != 0}).second)
      return jfail(FQ3_ERR_INVALID, "segment pushed twice in one call");
    off += lens[i];
  }
  return 0;
}

// the uniform plan of fq3_join_create / fq3_join_reset: [0, P, ..., P, 0]
int uniform(int32_t n_segments, int32_t pause_ms, std::vector<int32_t>* plan) {
  if (n_segments < 1) return jfail(FQ3_ERR_INVALID, "a join needs at least one segment");
  if (pause_ms < 0 || pause_ms > FQ3_JOIN_PAUSE_MAX_MS) return jfail(FQ3_ERR_INVALID, "pause_ms must be in [0, 2000]");
  plan->assign(n_segments + 1, pause_ms);
  plan->front() = plan->back() = 0;
  return 0;
}

// a new request of n_segments with the plan pauses_ms[0 .. n_segments]; frees what the join still held
int start(fq3_join* j, int32_t n_segments, const int32_t* pauses_ms) {
  if (n_segments < 1) return jfail(FQ3_ERR_INVALID, "a join needs at least one segment");
  if (!pauses_ms) return jfail(FQ3_ERR_INVALID, "null argument");
  for (int k = 0; k <= n_segments; ++k)
    if (pauses_ms[k] < 0 || pauses_ms[k] > FQ3_JOIN_BREAK_MAX_MS)
      return jfail(FQ3_ERR_INVALID, "every pause must be in [0, 10000] ms");
  free_chunks(j);
  j->S = n_segments;
  j->pause.resize(n_segments + 1);
  for (int k = 0; k <= n_segments; ++k) j->pause[k] = (int64_t)pauses_ms[k] * (FQ3_JOIN_RATE / 1000);
  j->cur = j->pp = 0;
  j->out_pos = j->released = 0;
  j->lead_done = j->tail_done = false;
  j->segs.assign(n_segments, Seg());
  return 0;
}

}  // namespace

extern "C" int fq3_join_create_pauses(int32_t device, int32_t n_segments, const int32_t* pauses_ms, fq3_join** out) {
  if (!out) return jfail(FQ3_ERR_INVALID, "null argument");
  DevGuard g(device);
  fq3_join* j = new fq3_join();
  j->dev = device;
  if (int rc = start(j, n_segments, pauses_ms)) {
    delete j;
    return rc;
  }
  if (cudaMalloc(&j->tail, 2 * F * sizeof(float)) != cudaSuccess) {
    delete j;
    return jfail(FQ3_ERR_CUDA, "cudaMalloc of the join tail failed");
  }
  *out = j;
  return 0;
}

extern "C" int fq3_join_create(int32_t device, int32_t n_segments, int32_t pause_ms, fq3_join** out) {
  std::vector<int32_t> plan;
  if (int rc = uniform(n_segments, pause_ms, &plan)) return rc;
  return fq3_join_create_pauses(device, n_segments, plan.data(), out);
}

extern "C" int fq3_join_reset_pauses(fq3_join* j, int32_t n_segments, const int32_t* pauses_ms) {
  if (!j) return jfail(FQ3_ERR_INVALID, "null argument");
  DevGuard g(j->dev);
  return start(j, n_segments, pauses_ms);
}

extern "C" int fq3_join_reset(fq3_join* j, int32_t n_segments, int32_t pause_ms) {
  std::vector<int32_t> plan;
  if (int rc = uniform(n_segments, pause_ms, &plan)) return rc;
  return fq3_join_reset_pauses(j, n_segments, plan.data());
}

extern "C" void fq3_join_destroy(fq3_join* j) {
  if (!j) return;
  DevGuard g(j->dev);
  free_chunks(j);
  cudaFree(j->tail);
  delete j;
}

extern "C" int fq3_join_released(fq3_join* const* joins, int32_t n_joins, int32_t n_pushes, const int32_t* join_of,
                                 const int32_t* seg, const int64_t* lens, const int32_t* ends, int64_t* released) {
  std::vector<std::map<int, Push>> per;
  if (int rc = group(joins, n_joins, n_pushes, join_of, seg, lens, ends, &per)) return rc;
  if (!released) return jfail(FQ3_ERR_INVALID, "null argument");
  for (int b = 0; b < n_joins; ++b)
    if (int rc = plan(joins[b], per[b], false, nullptr, nullptr, &released[b], nullptr, nullptr, nullptr)) return rc;
  return 0;
}

extern "C" int64_t fq3_join_total(const fq3_join* j) { return j ? j->released : -1; }

extern "C" int fq3_join_process(fq3_join* const* joins, int32_t n_joins, int32_t n_pushes, const int32_t* join_of,
                                const int32_t* seg, const int64_t* lens, const int32_t* ends, const float* in_dev,
                                float* out_dev, int64_t out_cap, void* stream_) {
  std::vector<std::map<int, Push>> per;
  if (int rc = group(joins, n_joins, n_pushes, join_of, seg, lens, ends, &per)) return rc;
  if (((uintptr_t)in_dev | (uintptr_t)out_dev) & 3) return jfail(FQ3_ERR_INVALID, "misaligned buffer");
  std::vector<int64_t> counts(n_joins);
  int64_t need = 0, in_total = 0;
  for (int b = 0; b < n_joins; ++b) {   // every refusal before anything is allocated or launched
    if (int rc = plan(joins[b], per[b], false, nullptr, nullptr, &counts[b], nullptr, nullptr, nullptr)) return rc;
    need += counts[b];
  }
  for (int i = 0; i < n_pushes; ++i) in_total += lens[i];
  if (in_total > 0 && !in_dev) return jfail(FQ3_ERR_INVALID, "null input buffer");
  if (need > 0 && !out_dev) return jfail(FQ3_ERR_INVALID, "null output buffer");
  if (need > out_cap) return jfail(FQ3_ERR_INVALID, "output buffer smaller than the released samples");
  DevGuard g(joins[0]->dev);
  cudaStream_t stream = (cudaStream_t)stream_;
  std::vector<Piece> pieces;
  std::vector<float*> to_free;
  int64_t off = 0;
  for (int b = 0; b < n_joins; ++b) {
    if (int rc = plan(joins[b], per[b], true, in_dev, out_dev + off, nullptr, &pieces, &to_free, stream)) return rc;
    off += counts[b];
  }
  cudaError_t e = cudaSuccess;
  if (!pieces.empty()) {
    Piece* d = nullptr;
    e = cudaMallocAsync(&d, sizeof(Piece) * pieces.size(), stream);
    if (e == cudaSuccess)
      e = cudaMemcpyAsync(d, pieces.data(), sizeof(Piece) * pieces.size(), cudaMemcpyHostToDevice, stream);
    if (e == cudaSuccess) {
      static const Fade fade = make_fade();
      join_kernel<<<(unsigned)pieces.size(), THREADS, 0, stream>>>(d, fade);
      e = cudaGetLastError();
    }
    if (d) cudaFreeAsync(d, stream);
  }
  for (float* p : to_free) cudaFreeAsync(p, stream);
  if (e != cudaSuccess) return jfail(FQ3_ERR_CUDA, cudaGetErrorString(e));
  return 0;
}

extern "C" const char* fq3_join_last_error(void) { return g_jerr; }
