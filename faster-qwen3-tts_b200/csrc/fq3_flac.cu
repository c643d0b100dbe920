// fq3_flac.cu -- FLAC output: lossless compression of s16 PCM that is already on the device (the resampler's s16
// store), for any number of streams in one launch.  The format and every encoder decision are fixed exactly
// (DESIGN.md, "FLAC output"; faster_qwen3_tts/flac.py states them, oracle/flac_oracle.py restates them in numpy):
//
//   stream  = "fLaC", STREAMINFO (last block): min/max block 16/4096, frame sizes 0, rate, mono, 16 bits, total samples
//             (0 unless the push that releases the header also flushes), MD5 0.
//   blocks  = variable blocking: a push of m samples after c carried ones encodes 16 floor((c + m) / 16) of them (all
//             at flush) as blocks of 4096 and one of the remainder; the rest (< 16) carries to the next push.
//   header  = sync 0xFFF9, block-size code 12 (4096) / 6 (8-bit n-1, n <= 256) / 7 (16-bit n-1), the rate's code, mono,
//             16 bits, the first sample's index (UTF-8 coded), CRC-8 (poly 0x07).
//   subframe = CONSTANT when all samples are equal; else the fewest-bit FIXED order o in 0 .. min(4, n-1), partition
//             order p in 0 .. 8 (n divisible by 2^p, n >> p > o), per partition the Rice parameter k in 0 .. 30 with
//             the fewest bits sum((u >> k) + 1 + k), u the zig-zag of the residual; method 0 when every k <= 14, else 1;
//             ties to the lowest o, then p, then k; VERBATIM when the best is not smaller.  No escapes, no wasted bits.
//   frame   = header, subframe, zero pad to a byte, CRC-16 (poly 0x8005) of everything before it.
//
// Output sizes depend on the data.  encode_kernel (one CTA per block) builds its frame in shared memory and stores it
// in a worst-case slot of a scratch buffer with its byte count; pack_kernel (one CTA per stream) then writes the stream
// header where one is due, the stream's frames back to back, and the new carry.  The host sizes every buffer by the
// bound fq3_flac_max_bytes and reads back one int32 byte count per stream.
//
// The choice is exact integer arithmetic.  encode_kernel forms, for each order in turn, the 64-bit sums F[j][k] of
// (u >> k) over the finest partitions the block allows (16 samples in a block of 4096); every coarser partition's cost
// for every k is a sum of those, and a shared 64-bit atomicMin over (cost << 5 | k) keeps the cheapest, lowest k.
// Bits are then placed with an exclusive scan of the code lengths and atomicOr into zeroed shared words (the unary
// zeros of a Rice code need no store), and the CRC-16 is the XOR of per-thread CRCs of 1/256th of the frame, each
// carried to the frame's end by a multiplication with x^(8 m) modulo the polynomial.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/fq3_engine.h"

namespace {

constexpr int THREADS = 256;
constexpr int NK = FQ3_FLAC_MAX_K + 1;                    // Rice parameters 0 .. 30
constexpr int NP = FQ3_FLAC_MAX_PARTITION_ORDER + 1;      // partition orders 0 .. 8
constexpr int NPART = (1 << NP) - 1;                      // (p, j) pairs: 511
constexpr int NORD = FQ3_FLAC_MAX_ORDER + 1;
constexpr int FRAME_HDR_MAX = 16;
constexpr int PER_THREAD = FQ3_FLAC_BLOCK / THREADS;    // samples of a block per thread in the partition sums
static_assert(PER_THREAD * THREADS == FQ3_FLAC_BLOCK, "a block is PER_THREAD samples per thread");

// shared layout of encode_kernel, in bytes
constexpr int SM_X = 0;                                            // int x[4096]
constexpr int SM_F = SM_X + FQ3_FLAC_BLOCK * 4;                    // u64 F[256][31]; later the frame words
constexpr int SM_BEST = SM_F + (1 << FQ3_FLAC_MAX_PARTITION_ORDER) * NK * 8;   // u64 best[511]
constexpr int SM_KB = SM_BEST + NPART * 8;                         // uint8 kb[5][511]
constexpr int SM_CAND = (SM_KB + NORD * NPART + 15) / 16 * 16;     // uint32 cand[5][9]
constexpr int SM_MISC = SM_CAND + NORD * NP * 4;                   // int misc[40]
constexpr int SMEM = SM_MISC + 40 * 4;
static_assert((2 * FQ3_FLAC_BLOCK + 19 + 8) <= (1 << FQ3_FLAC_MAX_PARTITION_ORDER) * NK * 8,
              "a frame fits in the F region");

thread_local char g_ferr[256] = "";
int ffail(int code, const char* msg) {
  snprintf(g_ferr, sizeof(g_ferr), "%s", msg);
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

int rate_code(int rate) {
  switch (rate) {
    case 8000: return 4;
    case 16000: return 5;
    case 22050: return 6;
    case 24000: return 7;
    case 32000: return 8;
    case 44100: return 9;
    case 48000: return 10;
    default: return -1;
  }
}

uint8_t crc8(const uint8_t* p, int n) {
  uint8_t c = 0;
  for (int i = 0; i < n; ++i) {
    c ^= p[i];
    for (int b = 0; b < 8; ++b) c = (uint8_t)((c & 0x80) ? (c << 1) ^ 0x07 : c << 1);
  }
  return c;
}

// the frame header of a block of n samples whose first sample has index `first`; returns its length
int frame_header(uint8_t* h, int n, int64_t first, int rate) {
  const int bs = n == FQ3_FLAC_BLOCK ? 12 : n <= 256 ? 6 : 7;
  int k = 0;
  h[k++] = 0xFF;
  h[k++] = 0xF9;   // sync, reserved 0, variable blocking
  h[k++] = (uint8_t)((bs << 4) | rate_code(rate));
  h[k++] = 0x08;   // mono, 16 bits
  const uint64_t v = (uint64_t)first;
  if (v < 0x80) {
    h[k++] = (uint8_t)v;
  } else {
    int nb = 2;
    while (nb < 7 && v >= (1ull << (5 * nb + 1))) ++nb;   // 2 bytes hold 11 bits, 3 hold 16, ... 6 hold 31, 7 hold 36
    h[k++] = nb == 7 ? 0xFE : (uint8_t)(((0xFF << (8 - nb)) & 0xFF) | (v >> (6 * (nb - 1))));
    for (int i = nb - 2; i >= 0; --i) h[k++] = (uint8_t)(0x80 | ((v >> (6 * i)) & 0x3F));
  }
  if (bs == 6) {
    h[k++] = (uint8_t)(n - 1);
  } else if (bs == 7) {
    h[k++] = (uint8_t)((n - 1) >> 8);
    h[k++] = (uint8_t)(n - 1);
  }
  h[k] = crc8(h, k);
  return k + 1;
}

void stream_header(uint8_t* h, int rate, int64_t total) {
  memset(h, 0, FQ3_FLAC_HEAD_BYTES);
  memcpy(h, "fLaC", 4);
  h[4] = 0x80;   // last metadata block, STREAMINFO
  h[7] = 34;
  uint8_t* s = h + 8;
  s[0] = FQ3_FLAC_GRAIN >> 8;
  s[1] = FQ3_FLAC_GRAIN & 0xFF;
  s[2] = FQ3_FLAC_BLOCK >> 8;
  s[3] = FQ3_FLAC_BLOCK & 0xFF;
  // s[4 .. 9]: min / max frame size 0
  s[10] = (uint8_t)(rate >> 12);
  s[11] = (uint8_t)(rate >> 4);
  s[12] = (uint8_t)(((rate & 0xF) << 4) | (0 << 1) | (15 >> 4));   // rate, channels - 1, bps - 1 (high bit)
  s[13] = (uint8_t)(((15 & 0xF) << 4) | ((total >> 32) & 0xF));     // bps - 1 (low 4 bits), total (high 4 bits)
  s[14] = (uint8_t)(total >> 24);
  s[15] = (uint8_t)(total >> 16);
  s[16] = (uint8_t)(total >> 8);
  s[17] = (uint8_t)total;
  // s[18 .. 33]: MD5 unset
}

int64_t max_bytes(int64_t carried, int64_t n, bool flush) {
  const int64_t ready = carried + n;
  const int64_t take = flush ? ready : ready / FQ3_FLAC_GRAIN * FQ3_FLAC_GRAIN;
  const int64_t full = take / FQ3_FLAC_BLOCK, rest = take % FQ3_FLAC_BLOCK;
  return FQ3_FLAC_HEAD_BYTES + full * (2 * FQ3_FLAC_BLOCK + 19) + (rest ? 2 * rest + 19 : 0);
}

struct Blk {                 // one frame
  const int16_t* carry;      // the stream's carried samples: seq[0, c)
  const int16_t* in;         // its new samples: seq[c, ...)
  unsigned char* slot;       // worst-case slot in the scratch buffer
  int* size;                 // <- the frame's bytes
  int c, start, n, hlen;     // the block is seq[start, start + n)
  unsigned char hdr[FRAME_HDR_MAX];
};

struct Pack {                // one stream
  const Blk* blks;           // its blocks, in order
  unsigned char* out;        // its output region
  int32_t* out_len;
  int16_t* carry;            // <- seq[take, take + rem)
  const int16_t* in;
  int nblk, c, take, rem, head;
  unsigned char hbytes[FQ3_FLAC_HEAD_BYTES];
};

__device__ __forceinline__ int residual(const int* x, int i, int o) {
  switch (o) {
    case 0: return x[i];
    case 1: return x[i] - x[i - 1];
    case 2: return x[i] - 2 * x[i - 1] + x[i - 2];
    case 3: return x[i] - 3 * x[i - 1] + 3 * x[i - 2] - x[i - 3];
    default: return x[i] - 4 * x[i - 1] + 6 * x[i - 2] - 4 * x[i - 3] + x[i - 4];
  }
}

__device__ __forceinline__ uint32_t zigzag(int r) { return r >= 0 ? 2u * (uint32_t)r : 2u * (uint32_t)(-r) - 1u; }

// bits [pos, pos + nb) of the big-endian bit string held in W get v (nb <= 32; the bits must be zero before)
__device__ __forceinline__ void put_bits(uint32_t* W, uint32_t pos, uint32_t v, int nb) {
  if (nb == 0) return;
  const uint32_t w = pos >> 5, s = pos & 31;
  if (s + nb <= 32) {
    atomicOr(&W[w], v << (32 - s - nb));
  } else {
    const uint32_t hi = s + nb - 32;
    atomicOr(&W[w], v >> hi);
    atomicOr(&W[w + 1], v << (32 - hi));
  }
}

__device__ __forceinline__ uint32_t byte_at(const uint32_t* W, int b) { return (W[b >> 2] >> (24 - 8 * (b & 3))) & 0xFF; }

// a * b mod the CRC-16 polynomial x^16 + x^15 + x^2 + 1, over GF(2)
__device__ __forceinline__ uint32_t gf_mul(uint32_t a, uint32_t b) {
  uint32_t r = 0;
  for (int i = 15; i >= 0; --i) {
    r <<= 1;
    if (r & 0x10000) r ^= 0x18005;
    if ((b >> i) & 1) r ^= a;
  }
  return r;
}

// x^(8 m) mod the polynomial
__device__ uint32_t gf_xpow8(uint32_t m) {
  uint32_t r = 1, base = 0x100;
  while (m) {
    if (m & 1) r = gf_mul(r, base);
    base = gf_mul(base, base);
    m >>= 1;
  }
  return r;
}

__device__ __forceinline__ int block_exclusive_scan(int v, int* warp_sums, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = v;
  for (int d = 1; d < 32; d <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += t;
  }
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int w = 0; w < THREADS / 32; ++w) {
      const int t = warp_sums[w];
      warp_sums[w] = run;
      run += t;
    }
    *total = run;
  }
  __syncthreads();
  return warp_sums[warp] + incl - v;
}

__global__ void __launch_bounds__(THREADS) encode_kernel(const Blk* __restrict__ blks) {
  extern __shared__ __align__(16) unsigned char sm[];
  int* x = reinterpret_cast<int*>(sm + SM_X);
  unsigned long long* F = reinterpret_cast<unsigned long long*>(sm + SM_F);
  unsigned long long* best = reinterpret_cast<unsigned long long*>(sm + SM_BEST);
  unsigned char* kb = sm + SM_KB;
  uint32_t* cand = reinterpret_cast<uint32_t*>(sm + SM_CAND);
  int* misc = reinterpret_cast<int*>(sm + SM_MISC);   // [0] not constant, [1..3] choice, [4] total, [8..15] warps
  const Blk& B = blks[blockIdx.x];
  const int n = B.n, tid = threadIdx.x;
  if (tid == 0) misc[0] = 0;
  for (int i = tid; i < NORD * NP; i += THREADS) cand[i] = 0xFFFFFFFFu;
  __syncthreads();
  for (int i = tid; i < n; i += THREADS) {
    const int s = B.start + i;
    x[i] = s < B.c ? B.carry[s] : B.in[s - B.c];
  }
  __syncthreads();
  for (int i = tid; i < n; i += THREADS)
    if (x[i] != x[0]) misc[0] = 1;
  __syncthreads();
  const bool constant = misc[0] == 0;
  const int pmax = min(__ffs(n) - 1, FQ3_FLAC_MAX_PARTITION_ORDER);   // n divisible by 2^p for p <= pmax
  const int P = 1 << pmax, fsize = n >> pmax;
  if (!constant) {
    for (int o = 0; o <= min(FQ3_FLAC_MAX_ORDER, n - 1); ++o) {
      // F[j][k] = sum of (u >> k) over the residuals of finest partition j: each thread sums its PER_THREAD samples in
      // registers (u < 2^20) and adds them to F when its samples leave a partition
      for (int i = tid; i < P * NK; i += THREADS) F[i] = 0;
      for (int i = tid; i < NPART; i += THREADS) best[i] = ~0ull;
      __syncthreads();
      {
        uint32_t acc[NK];
        int cur = -1;
        for (int i = max(tid * PER_THREAD, o); i < min(tid * PER_THREAD + PER_THREAD, n); ++i) {
          const int j = i / fsize;
          if (j != cur) {
            if (cur >= 0) {
#pragma unroll
              for (int k = 0; k < NK; ++k)
                if (acc[k]) atomicAdd(&F[cur * NK + k], (unsigned long long)acc[k]);
            }
            cur = j;
#pragma unroll
            for (int k = 0; k < NK; ++k) acc[k] = 0;
          }
          const uint32_t u = zigzag(residual(x, i, o));
#pragma unroll
          for (int k = 0; k < NK; ++k) acc[k] += u >> k;
        }
        if (cur >= 0) {
#pragma unroll
          for (int k = 0; k < NK; ++k)
            if (acc[k]) atomicAdd(&F[cur * NK + k], (unsigned long long)acc[k]);
        }
      }
      __syncthreads();
      // every (p, j, k): the partition's cost, the cheapest (lowest k on ties) kept per (p, j).  k is the slowest
      // index, so the lanes of a warp update different (p, j) and the atomics do not contend within a warp
      int pairs = 0;
      for (int p = 0; p <= pmax; ++p)
        if ((n >> p) > o) pairs += 1 << p;
      for (int it = tid; it < pairs * NK; it += THREADS) {
        const int k = it / pairs;
        int p = 0, r = it - k * pairs;
        for (;; ++p) {
          if ((n >> p) <= o) continue;
          if (r < (1 << p)) break;
          r -= 1 << p;
        }
        const int j = r, span = 1 << (pmax - p);
        unsigned long long s = 0;
        for (int q = j * span; q < (j + 1) * span; ++q) s += F[q * NK + k];
        const uint64_t cnt = (uint64_t)((n >> p) - (j == 0 ? o : 0));
        const uint64_t cost = s + cnt * (uint64_t)(k + 1);
        atomicMin(&best[(1 << p) - 1 + j], (cost << 5) | (uint64_t)k);
      }
      __syncthreads();
      // per partition order: the residual section's bits, and each partition's k
      const int warp = tid >> 5, lane = tid & 31;
      for (int p = warp; p <= pmax; p += THREADS / 32) {
        if ((n >> p) <= o) continue;
        uint32_t bits = 0, kmax = 0;
        for (int j = lane; j < (1 << p); j += 32) {
          const unsigned long long b = best[(1 << p) - 1 + j];
          const uint32_t k = (uint32_t)(b & 31);
          bits += (uint32_t)(b >> 5);
          kmax = max(kmax, k);
          kb[o * NPART + (1 << p) - 1 + j] = (unsigned char)k;
        }
        for (int d = 16; d; d >>= 1) {
          bits += __shfl_xor_sync(0xffffffffu, bits, d);
          kmax = max(kmax, __shfl_xor_sync(0xffffffffu, kmax, d));
        }
        if (lane == 0) cand[o * NP + p] = 8 + 16 * o + 6 + (1u << p) * (kmax > 14 ? 5 : 4) + bits;
      }
      __syncthreads();
    }
    if (tid == 0) {
      uint32_t bb = 0xFFFFFFFFu;
      int bo = -1, bp = -1;
      for (int o = 0; o < NORD; ++o)
        for (int p = 0; p < NP; ++p)
          if (cand[o * NP + p] < bb) bb = cand[o * NP + p], bo = o, bp = p;
      if (bo < 0 || bb >= 8u + 16u * (uint32_t)n) bo = -1;   // VERBATIM
      misc[1] = bo;
      misc[2] = bp;
      int method = 0;
      if (bo >= 0)
        for (int j = 0; j < (1 << bp); ++j) method |= kb[bo * NPART + (1 << bp) - 1 + j] > 14;
      misc[3] = method;
    }
  }
  // the frame, in big-endian bit order, in zeroed shared words over the F region
  uint32_t* W = reinterpret_cast<uint32_t*>(F);
  const int nwords = (FRAME_HDR_MAX + 1 + 2 * n + 2 + 3) / 4 + 1;
  for (int i = tid; i < nwords; i += THREADS) W[i] = 0;
  __syncthreads();
  const int o = constant ? -2 : misc[1], p = misc[2], method = misc[3];
  for (int i = tid; i < B.hlen; i += THREADS) put_bits(W, 8 * i, B.hdr[i], 8);
  uint32_t pos = 8 * B.hlen;
  uint32_t end;
  if (o == -2) {   // CONSTANT
    if (tid == 0) {
      put_bits(W, pos, 0x00, 8);
      put_bits(W, pos + 8, (uint32_t)x[0] & 0xFFFF, 16);
    }
    end = pos + 24;
  } else if (o == -1) {   // VERBATIM
    if (tid == 0) put_bits(W, pos, 0x02, 8);
    for (int i = tid; i < n; i += THREADS) put_bits(W, pos + 8 + 16 * i, (uint32_t)x[i] & 0xFFFF, 16);
    end = pos + 8 + 16 * n;
  } else {   // FIXED
    if (tid == 0) {
      put_bits(W, pos, (uint32_t)((0x08 | o) << 1), 8);
      put_bits(W, pos + 8 + 16 * o, (uint32_t)((method << 4) | p), 6);
    }
    for (int i = tid; i < o; i += THREADS) put_bits(W, pos + 8 + 16 * i, (uint32_t)x[i] & 0xFFFF, 16);
    pos += 8 + 16 * o + 6;
    const int psize = n >> p, w = 4 + method, cnt = n - o;
    const unsigned char* ks = kb + o * NPART + (1 << p) - 1;
    const int per = (cnt + THREADS - 1) / THREADS;
    const int i0 = o + tid * per, i1 = min(o + (tid + 1) * per, n);
    int mine = 0;
    for (int i = i0; i < i1; ++i) {
      const int j = i / psize, k = ks[j];
      const bool first = i == (j == 0 ? o : j * psize);
      mine += (first ? w : 0) + (int)(zigzag(residual(x, i, o)) >> k) + 1 + k;
    }
    int total;
    int off = block_exclusive_scan(mine, misc + 8, misc + 4);
    total = misc[4];
    for (int i = i0; i < i1; ++i) {
      const int j = i / psize, k = ks[j];
      const uint32_t u = zigzag(residual(x, i, o));
      uint32_t at = pos + off;
      if (i == (j == 0 ? o : j * psize)) {
        put_bits(W, at, (uint32_t)k, w);
        at += w;
      }
      const uint32_t q = u >> k;
      put_bits(W, at + q, (1u << k) | (u & ((1u << k) - 1)), k + 1);
      off += (int)(at - (pos + off)) + (int)q + 1 + k;
    }
    end = pos + total;
  }
  __syncthreads();
  // CRC-16 of bytes [0, len): per thread a CRC of its share, carried to the end by x^(8 m)
  const int len = (int)((end + 7) >> 3);
  const int share = (len + THREADS - 1) / THREADS;
  const int b0 = min(tid * share, len), b1 = min(b0 + share, len);
  uint32_t crc = 0;
  for (int b = b0; b < b1; ++b) {
    crc ^= byte_at(W, b) << 8;
    for (int r = 0; r < 8; ++r) crc = (crc & 0x8000) ? ((crc << 1) ^ 0x8005) & 0xFFFF : (crc << 1) & 0xFFFF;
  }
  if (crc && b1 < len) crc = gf_mul(crc, gf_xpow8((uint32_t)(len - b1)));
  for (int d = 16; d; d >>= 1) crc ^= __shfl_xor_sync(0xffffffffu, crc, d);
  __syncthreads();   // every thread has read W before the CRC lands in it
  if ((tid & 31) == 0) misc[16 + (tid >> 5)] = (int)crc;
  __syncthreads();
  if (tid == 0) {
    uint32_t c = 0;
    for (int wi = 0; wi < THREADS / 32; ++wi) c ^= (uint32_t)misc[16 + wi];
    put_bits(W, 8 * len, c, 16);
    *B.size = len + 2;
  }
  __syncthreads();
  for (int b = tid; b < len + 2; b += THREADS) B.slot[b] = (unsigned char)byte_at(W, b);
}

__global__ void __launch_bounds__(THREADS) pack_kernel(const Pack* __restrict__ packs) {
  const Pack& S = packs[blockIdx.x];
  const int tid = threadIdx.x;
  int off = 0;
  if (S.head) {
    for (int i = tid; i < FQ3_FLAC_HEAD_BYTES; i += THREADS) S.out[i] = S.hbytes[i];
    off = FQ3_FLAC_HEAD_BYTES;
  }
  for (int b = 0; b < S.nblk; ++b) {
    const Blk& B = S.blks[b];
    const int sz = *B.size;
    for (int i = tid; i < sz; i += THREADS) S.out[off + i] = B.slot[i];
    off += sz;
  }
  // the new carry, seq[take, take + rem): with take == 0 it is the old carry (read and written by the same thread)
  // followed by new samples; with take > 0 it comes from the new samples alone
  for (int i = tid; i < S.rem; i += THREADS) {
    const int s = S.take + i;
    S.carry[i] = s < S.c ? S.carry[s] : S.in[s - S.c];
  }
  if (tid == 0) *S.out_len = off;
}

}  // namespace

struct fq3_flac {
  int dev = 0, rate = 0;
  int64_t index = 0;     // samples encoded so far: the index of the first carried sample
  int carried = 0;
  bool started = false, flushed = false;
  int16_t* carry = nullptr;
};

extern "C" int fq3_flac_create(int32_t device, int32_t rate, fq3_flac** out) {
  if (!out) return ffail(FQ3_ERR_INVALID, "null argument");
  if (rate_code(rate) < 0)
    return ffail(FQ3_ERR_INVALID, "FLAC rate must be one of 8000, 16000, 22050, 24000, 32000, 44100, 48000");
  DevGuard g(device);
  fq3_flac* f = new fq3_flac();
  f->dev = device;
  f->rate = rate;
  if (cudaMalloc(&f->carry, FQ3_FLAC_GRAIN * sizeof(int16_t)) != cudaSuccess) {
    delete f;
    return ffail(FQ3_ERR_CUDA, "cudaMalloc of the FLAC carry failed");
  }
  *out = f;
  return 0;
}

extern "C" int fq3_flac_reset(fq3_flac* f) {
  if (!f) return ffail(FQ3_ERR_INVALID, "null argument");
  f->index = 0;
  f->carried = 0;
  f->started = f->flushed = false;
  return 0;
}

extern "C" void fq3_flac_destroy(fq3_flac* f) {
  if (!f) return;
  DevGuard g(f->dev);
  cudaFree(f->carry);
  delete f;
}

extern "C" int64_t fq3_flac_max_bytes(int64_t carried, int64_t n, int32_t flush) {
  if (carried < 0 || carried >= FQ3_FLAC_GRAIN || n < 0) return -1;
  return max_bytes(carried, n, flush != 0);
}

extern "C" int fq3_flac_process(fq3_flac* const* encs, int32_t n_streams, const int16_t* in_dev,
                                const int64_t* in_lens, const int32_t* flush, void* out_dev, int64_t out_cap,
                                int32_t* out_lens_dev, void* stream_) {
  if (!encs || n_streams <= 0 || !in_lens || !flush) return ffail(FQ3_ERR_INVALID, "null argument");
  if (!out_lens_dev) return ffail(FQ3_ERR_INVALID, "null output length buffer");
  if ((uintptr_t)in_dev & 1) return ffail(FQ3_ERR_INVALID, "misaligned input buffer (int16 needs 2-byte alignment)");
  if ((uintptr_t)out_dev & (FQ3_FLAC_ALIGN - 1))
    return ffail(FQ3_ERR_INVALID, "misaligned output buffer (each stream's region starts 16-byte aligned)");
  if ((uintptr_t)out_lens_dev & 3) return ffail(FQ3_ERR_INVALID, "misaligned output length buffer");
  const int dev = encs[0] ? encs[0]->dev : 0;
  std::vector<Blk> blks;
  std::vector<Pack> packs(n_streams);
  std::vector<int> first_blk(n_streams);
  std::vector<int64_t> slot_off;
  int64_t in_off = 0, out_off = 0, scratch = 0;
  for (int b = 0; b < n_streams; ++b) {
    fq3_flac* f = encs[b];
    if (!f) return ffail(FQ3_ERR_INVALID, "null FLAC encoder handle");
    if (f->dev != dev) return ffail(FQ3_ERR_INVALID, "FLAC encoder handles of different devices");
    for (int a = 0; a < b; ++a)
      if (encs[a] == f) return ffail(FQ3_ERR_INVALID, "FLAC encoder listed twice");
    if (f->flushed) return ffail(FQ3_ERR_STATE, "FLAC encoder already flushed (reset it to start a new stream)");
    if (in_lens[b] < 0) return ffail(FQ3_ERR_INVALID, "negative input length");
    const bool fl = flush[b] != 0;
    const int64_t ready = f->carried + in_lens[b];
    const int64_t take = fl ? ready : ready / FQ3_FLAC_GRAIN * FQ3_FLAC_GRAIN;
    if (f->index + ready >= (1ll << 36)) return ffail(FQ3_ERR_INVALID, "FLAC stream longer than 2^36 samples");
    Pack& P = packs[b];
    out_off = (out_off + FQ3_FLAC_ALIGN - 1) / FQ3_FLAC_ALIGN * FQ3_FLAC_ALIGN;
    P.out = (unsigned char*)out_dev + out_off;
    out_off += max_bytes(f->carried, in_lens[b], fl);
    P.out_len = out_lens_dev + b;
    P.carry = f->carry;
    P.in = in_dev + in_off;
    P.c = f->carried;
    P.take = (int)take;
    P.rem = (int)(ready - take);
    P.head = !f->started;
    if (P.head) stream_header(P.hbytes, f->rate, fl ? f->index + ready : 0);
    first_blk[b] = (int)blks.size();
    for (int64_t s0 = 0; s0 < take; s0 += FQ3_FLAC_BLOCK) {
      Blk B{};
      B.carry = f->carry;
      B.in = in_dev + in_off;
      B.c = f->carried;
      B.start = (int)s0;
      B.n = (int)std::min<int64_t>(FQ3_FLAC_BLOCK, take - s0);
      B.hlen = frame_header(B.hdr, B.n, f->index + s0, f->rate);
      slot_off.push_back(scratch);
      scratch += (2 * B.n + 19 + 15) / 16 * 16;
      blks.push_back(B);
    }
    P.nblk = (int)blks.size() - first_blk[b];
    in_off += in_lens[b];
  }
  if (in_off > 0 && !in_dev) return ffail(FQ3_ERR_INVALID, "null input buffer");
  if (!out_dev) return ffail(FQ3_ERR_INVALID, "null output buffer");
  if (out_off > out_cap) return ffail(FQ3_ERR_INVALID, "output buffer smaller than the bound of the released bytes");
  if (in_off >= (1ll << 31)) return ffail(FQ3_ERR_INVALID, "push longer than 2^31 samples");
  {
    DevGuard g(dev);
    cudaStream_t stream = (cudaStream_t)stream_;
    // blocks, packs, frame sizes and frame slots in one stream-ordered allocation
    const size_t nb = blks.size();
    const size_t bb = sizeof(Blk) * nb, pb = sizeof(Pack) * n_streams, sb = (sizeof(int) * nb + 15) / 16 * 16;
    const size_t head = (bb + pb + sb + 15) / 16 * 16;
    void* d = nullptr;
    cudaError_t e = cudaMallocAsync(&d, head + (size_t)scratch, stream);
    if (e == cudaSuccess) {
      unsigned char* base = (unsigned char*)d;
      Blk* dblk = (Blk*)base;
      int* dsize = (int*)(base + bb + pb);
      for (size_t i = 0; i < nb; ++i) {
        blks[i].slot = base + head + slot_off[i];
        blks[i].size = dsize + i;
      }
      for (int b = 0; b < n_streams; ++b) packs[b].blks = dblk + first_blk[b];
      std::vector<unsigned char> blob(bb + pb);
      memcpy(blob.data(), blks.data(), bb);
      memcpy(blob.data() + bb, packs.data(), pb);
      e = cudaMemcpyAsync(d, blob.data(), blob.size(), cudaMemcpyHostToDevice, stream);
      if (e == cudaSuccess && nb)
        e = cudaFuncSetAttribute(encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
      if (e == cudaSuccess && nb) {
        encode_kernel<<<(unsigned)nb, THREADS, SMEM, stream>>>(dblk);
        e = cudaGetLastError();
      }
      if (e == cudaSuccess) {
        pack_kernel<<<(unsigned)n_streams, THREADS, 0, stream>>>((const Pack*)(base + bb));
        e = cudaGetLastError();
      }
    }
    if (d) cudaFreeAsync(d, stream);
    if (e != cudaSuccess) return ffail(FQ3_ERR_CUDA, cudaGetErrorString(e));
  }
  for (int b = 0; b < n_streams; ++b) {
    fq3_flac* f = encs[b];
    const Pack& P = packs[b];
    f->index += P.take;
    f->carried = P.rem;
    f->started = true;
    f->flushed = flush[b] != 0;
  }
  return 0;
}

extern "C" const char* fq3_flac_last_error(void) { return g_ferr; }
