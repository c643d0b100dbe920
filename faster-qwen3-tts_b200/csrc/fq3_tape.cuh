// fq3_tape.cuh -- the weight tape (DESIGN §3): every GEMV matrix (segment) of the decode program, repacked at load time
// into one slice per CTA in the order the CTA consumes it.  A slice holds, segment by segment, the CTA's row groups; a
// group is ntiles tiles of at most STAGE_BYTES (one ring stage each), in the fp32 layout (rows x 512-byte row chunks) or
// the bf16 one (m-tiles x 2048-byte k-groups of mma.m16n8k16 A fragments, pack_mma_kernel).  Kinds of a bf16 group:
// FULL (16 rows per m-tile), HALF (8 rows, their two K halves in one m-tile), GU (8 gate/up row pairs per m-tile).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/fq3_engine.h"

namespace fq3 {

constexpr int STAGE_BYTES = 32768;   // one ring stage: the largest tile
constexpr int MAXGRP = 512;          // row groups per CTA
constexpr int MAXSEG = 256;          // GEMV segments

struct Grp {           // one row group of one segment, as seen by one CTA (full K)
  uint32_t off16;      // tape offset / 16
  int32_t row0;        // first row inside the segment (bf16 GU: first gate/up pair)
  uint16_t rows;       // fp32: row count (even, <= 32); bf16: n_mt | kind << 8 (grp_nmt, grp_kind)
  uint16_t m;          // K-chunks per tile: fp32 512-byte row chunks, bf16 k-groups G
  uint16_t ntiles;     // tiles: m * ntiles chunks cover K (bf16 HALF: K / 2)
  uint16_t pad;
};

enum GrpKind { GRP_FULL = 0, GRP_HALF = 1, GRP_GU = 2 };

// bf16 group header: m-tiles and kind (Grp::rows, PackGrp::rows)
__host__ __device__ __forceinline__ int grp_nmt(uint16_t rows) { return rows & 0xff; }
__host__ __device__ __forceinline__ int grp_kind(uint16_t rows) { return rows >> 8; }
// bytes of one tile of a group with header rows / m
__host__ __device__ __forceinline__ uint32_t tile_bytes(bool bf16, uint16_t rows, uint16_t m) {
  return bf16 ? (uint32_t)(rows & 0xff) * m * 2048u : (uint32_t)rows * m * 512u;
}
// segment table word [cta][seg]: this CTA's groups of the segment are grp[begin .. begin + n) (begin relative to the
// CTA's first group)
__host__ __device__ __forceinline__ int seg_begin(uint32_t st) { return (int)(st >> 8); }
__host__ __device__ __forceinline__ int seg_count(uint32_t st) { return (int)(st & 255u); }

// ---- pack kernels: one block per group record, rowsrc[rowsrc_idx + r] = address of the group's r-th source row
struct PackGrp {
  uint64_t tape_off;
  uint32_t rowsrc_idx;
  uint16_t rows, m, ntiles, pad;   // as Grp
  int32_t K;
};

__global__ void pack_kernel(const PackGrp* __restrict__ pg, int npg, const void* const* __restrict__ rowsrc,
                            uint8_t* __restrict__ tape) {
  for (int b = blockIdx.x; b < npg; b += gridDim.x) {
    const PackGrp g = pg[b];
    const int rows = g.rows, m = g.m;
    const long long total = (long long)rows * m * g.ntiles * 32;
    uint4* dst = reinterpret_cast<uint4*>(tape + g.tape_off);
    for (long long q = threadIdx.x; q < total; q += blockDim.x) {
      const int lane = (int)(q & 31);
      long long rem = q >> 5;
      const int j = (int)(rem % m);
      rem /= m;
      const int r = (int)(rem % rows);
      const int t = (int)(rem / rows);
      const int kb = t * m + j;
      const uint8_t* src = reinterpret_cast<const uint8_t*>(rowsrc[g.rowsrc_idx + r]);
      dst[q] = *reinterpret_cast<const uint4*>(src + ((size_t)kb * 128 + lane * 4) * 4);
    }
  }
}

// bf16 tensor-core layout: per tile [m-tile][k-group][step 0..3][lane][16 B] holding mma.m16n8k16 A fragments
// (a0,a1,a2,a3) = rowA[kk,kk+1], rowB[kkB,kkB+1], rowA[kk+2,kk+3], rowB[kkB+2,kkB+3], kk = 64*kgroup + 16*t + 4*step.
// kind 0 FULL: rowA = r0+16*mt+g, rowB = rowA+8;  kind 1 HALF: rowA = rowB = r0+g, kkB = K/2 + kk;
// kind 2 GU: rowA = gate row, rowB = up row of pair r0/2 + 8*mt + g (rowsrc holds gate/up interleaved).
__global__ void pack_mma_kernel(const PackGrp* __restrict__ pg, int npg, const void* const* __restrict__ rowsrc,
                                uint8_t* __restrict__ tape) {
  for (int b = blockIdx.x; b < npg; b += gridDim.x) {
    // header fields read one by one and 32-bit index arithmetic (a group holds ntiles * G <= K / 64 k-groups of at most
    // 2 m-tiles, far below 2^31 elements): with a struct copy and 64-bit division, ptxas for sm_90a took G from a
    // uniform register it never wrote, and the tape came out wrong
    const int n_mt = grp_nmt(pg[b].rows), kind = grp_kind(pg[b].rows), G = pg[b].m, ntiles = pg[b].ntiles, K = pg[b].K;
    const uint32_t rowsrc_idx = pg[b].rowsrc_idx;
    const int total = ntiles * n_mt * G * 128;
    uint4* dst = reinterpret_cast<uint4*>(tape + pg[b].tape_off);
    for (int q = threadIdx.x; q < total; q += blockDim.x) {
      const int lane = q & 31, st = (q >> 5) & 3;
      int rem = q >> 7;
      const int qq = rem % G;
      rem /= G;
      const int mt = rem % n_mt;
      const int tl = rem / n_mt;
      const int gq = lane >> 2, t = lane & 3;
      const int kk = 64 * (tl * G + qq) + 16 * t + 4 * st;
      const uint8_t *ra, *rb;
      int kb = kk;
      if (kind == 0) {
        ra = reinterpret_cast<const uint8_t*>(rowsrc[rowsrc_idx + mt * 16 + gq]);
        rb = reinterpret_cast<const uint8_t*>(rowsrc[rowsrc_idx + mt * 16 + gq + 8]);
      } else if (kind == 1) {
        ra = rb = reinterpret_cast<const uint8_t*>(rowsrc[rowsrc_idx + gq]);
        kb = K / 2 + kk;
      } else {
        ra = reinterpret_cast<const uint8_t*>(rowsrc[rowsrc_idx + 2 * (mt * 8 + gq)]);
        rb = reinterpret_cast<const uint8_t*>(rowsrc[rowsrc_idx + 2 * (mt * 8 + gq) + 1]);
      }
      const uint2 a = *reinterpret_cast<const uint2*>(ra + (size_t)kk * 2);
      const uint2 c = *reinterpret_cast<const uint2*>(rb + (size_t)kb * 2);
      dst[q] = make_uint4(a.x, c.x, a.y, c.y);
    }
  }
}

// ---- segments: the GEMV matrices of the decode program, in tape order
struct TapeRun {       // rows [row0, row0 + rows) of the row-major [tensor_rows][K] weight `tensor`
  std::string tensor;
  int64_t tensor_rows, row0, rows;
};
struct TapeSeg {
  int rows, K;
  bool gu;             // gate/up: runs = {gate, up}, and the segment's rows interleave them (2p = gate p, 2p + 1 = up p)
  std::vector<TapeRun> runs;   // otherwise the rows of the runs one after the other
};
struct TapeSegments {
  std::vector<TapeSeg> segs;
  // [0] talker, [1] predictor: layer l uses seg_base + 4*l + {0:QKV, 1:O, 2:GU, 3:DN}; the talker has one head
  // segment, the predictor one per code group from seg_head on.  seg_mtp = -1 without the MTP projection.
  int seg_base[2], seg_head[2], seg_mtp;
};

// talker layers, talker head, predictor layers, predictor heads, MTP projection
inline TapeSegments tape_segments(const fq3_config& cfg) {
  TapeSegments T;
  auto seg = [&](int64_t rows, int64_t K, bool gu, std::vector<TapeRun> runs) {
    T.segs.push_back(TapeSeg{(int)rows, (int)K, gu, std::move(runs)});
  };
  for (int si = 0; si < 2; ++si) {
    const fq3_stack_config& c = si == 0 ? cfg.talker : cfg.predictor;
    const std::string p = si == 0 ? "t." : "p.";
    const int64_t L = c.num_hidden_layers, H = c.hidden_size, I = c.intermediate_size, V = c.vocab_size;
    const int64_t qd = c.num_attention_heads * 128, kd = c.num_key_value_heads * 128;
    T.seg_base[si] = (int)T.segs.size();
    for (int64_t l = 0; l < L; ++l) {
      seg(qd + 2 * kd, H, false, {{p + "q", L * qd, l * qd, qd}, {p + "k", L * kd, l * kd, kd}, {p + "v", L * kd, l * kd, kd}});
      seg(H, qd, false, {{p + "o", L * H, l * H, H}});
      seg(2 * I, H, true, {{p + "gate", L * I, l * I, I}, {p + "up", L * I, l * I, I}});
      seg(H, I, false, {{p + "down", L * H, l * H, H}});
    }
    T.seg_head[si] = (int)T.segs.size();
    const int64_t nh = si == 0 ? 1 : cfg.num_code_groups - 1;
    for (int64_t i = 0; i < nh; ++i) seg(V, H, false, {{si == 0 ? "t.head" : "p.heads", nh * V, i * V, V}});
  }
  T.seg_mtp = cfg.has_mtp_projection ? (int)T.segs.size() : -1;
  const int64_t Hp = cfg.predictor.hidden_size, Ht = cfg.talker.hidden_size;
  if (cfg.has_mtp_projection) seg(Hp, Ht, false, {{"p.mtp_w", Hp, 0, Hp}});
  return T;
}

// append the addresses of segment s's rows to the row-source table; w[i] is the device address of s.runs[i].tensor
inline void tape_rows(const TapeSeg& s, const void* const* w, size_t esz, std::vector<const void*>& rowsrc) {
  auto row = [&](size_t i, int64_t r) -> const void* {
    return (const uint8_t*)w[i] + (size_t)(s.runs[i].row0 + r) * s.K * esz;
  };
  for (int64_t p = 0; s.gu && p < s.rows / 2; ++p) {
    rowsrc.push_back(row(0, p));
    rowsrc.push_back(row(1, p));
  }
  for (size_t i = 0; !s.gu && i < s.runs.size(); ++i)
    for (int64_t r = 0; r < s.runs[i].rows; ++r) rowsrc.push_back(row(i, r));
}

// ---- planner: which rows of each segment every CTA streams, as row groups, and where they sit on the tape
struct TapePlan {
  std::vector<Grp> grps;              // CTA-major, consumption order, off16 set
  std::vector<uint32_t> segtab;       // [ncta][nseg] seg_begin / seg_count words
  std::vector<uint32_t> cta_grp_off;  // [ncta + 1]: CTA c's groups are grps[cta_grp_off[c] .. cta_grp_off[c + 1])
  std::vector<PackGrp> pack;          // pack record of grps[i]
  uint64_t tape_bytes = 0;
};

// the largest divisor of n that is at most cap (1 if none is)
inline int largest_divisor(int n, int cap) {
  int r = 1;
  for (int d = 1; d <= n; ++d)
    if (n % d == 0 && d <= cap) r = d;
  return r;
}

// A segment is dealt out in whole units (bf16: 8 rows, or 8 gate/up pairs; fp32: a row pair), base or base + 1 per CTA;
// the `extra` larger shares rotate on from segment to segment so that no CTA takes every remainder.  A CTA's units
// become row groups of at most 32 rows (bf16: up to 2 m-tiles of one kind), each tiled with the largest divisor of its
// K-chunks that keeps a tile within STAGE_BYTES.  Returns "" or the refusal.
inline std::string plan_tape(const std::vector<TapeSeg>& segs, int ncta, bool bf16, TapePlan& plan) {
  const int nseg = (int)segs.size();
  if (nseg > MAXSEG) return "too many segments (" + std::to_string(nseg) + " > " + std::to_string(MAXSEG) + ")";
  plan = TapePlan();
  std::vector<std::vector<Grp>> cta_grps(ncta);
  std::vector<uint32_t>& segtab = plan.segtab;
  segtab.assign((size_t)ncta * nseg, 0);
  std::vector<uint32_t> rowsrc0(nseg + 1, 0);   // first row-source index of each segment
  int rot = 0;
  for (int sg = 0; sg < nseg; ++sg) {
    const int rows = segs[sg].rows, K = segs[sg].K;
    rowsrc0[sg + 1] = rowsrc0[sg] + (uint32_t)rows;
    const int unit_rows = bf16 ? (segs[sg].gu ? 16 : 8) : 2;
    const std::string at = "segment " + std::to_string(sg) + ": rows " + std::to_string(rows);
    if (rows % unit_rows || K % 128)
      return at + (bf16 ? " / K " + std::to_string(K) + " not tileable for the bf16 tensor-core tape"
                        : " must be even and K " + std::to_string(K) + " a multiple of 128");
    const int units = rows / unit_rows, base = units / ncta, extra = units % ncta;
    int unit0 = 0;
    for (int c = 0; c < ncta; ++c) {
      const int uc = base + ((((c - rot) % ncta + ncta) % ncta) < extra ? 1 : 0);
      std::vector<Grp>& cg = cta_grps[c];
      const int begin = (int)cg.size();
      // header rows / m, first row row0: K-chunks are 64-column k-groups (HALF: of K / 2) or 128-element row chunks
      auto emit = [&](uint32_t hdr, int row0) {
        const int chunks = !bf16 ? K / 128 : grp_kind(hdr) == GRP_HALF ? K / 128 : K / 64;
        const int m = largest_divisor(chunks, STAGE_BYTES / (int)tile_bytes(bf16, hdr, 1));
        cg.push_back(Grp{0, row0, (uint16_t)hdr, (uint16_t)m, (uint16_t)(chunks / m), 0});
      };
      if (!bf16) {
        const int ng = (2 * uc + 31) / 32;
        for (int gi = 0, r0 = 2 * unit0; gi < ng; ++gi) {
          const int gr = 2 * (uc / ng + (gi < uc % ng ? 1 : 0));
          emit(gr, r0);
          r0 += gr;
        }
      } else if (segs[sg].gu) {
        for (int u = 0; u < uc; u += 2) emit(std::min(2, uc - u) | GRP_GU << 8, (unit0 + u) * 8);
      } else {
        const int nfull = uc / 2;
        for (int f = 0; f < nfull; f += 2) emit(std::min(2, nfull - f) | GRP_FULL << 8, (unit0 + 2 * f) * 8);
        if (uc % 2) emit(1 | GRP_HALF << 8, (unit0 + uc - 1) * 8);
      }
      const int ng = (int)cg.size() - begin;
      if (ng > 255) return "segment " + std::to_string(sg) + ": too many groups per CTA";
      segtab[(size_t)c * nseg + sg] = ((uint32_t)begin << 8) | (uint32_t)ng;
      unit0 += uc;
    }
    rot = (rot + extra) % ncta;
  }
  // lay the groups out CTA after CTA (each slice 1024-aligned), segment after segment within a CTA
  plan.cta_grp_off.assign(ncta + 1, 0);
  uint64_t off = 0;
  for (int c = 0; c < ncta; ++c) {
    for (int sg = 0; sg < nseg; ++sg) {
      const uint32_t st = segtab[(size_t)c * nseg + sg];
      for (int i = 0; i < seg_count(st); ++i) {
        Grp g = cta_grps[c][seg_begin(st) + i];
        g.off16 = (uint32_t)(off / 16);
        const uint32_t rsrc = rowsrc0[sg] + (uint32_t)(bf16 && grp_kind(g.rows) == GRP_GU ? 2 * g.row0 : g.row0);
        plan.grps.push_back(g);
        plan.pack.push_back(PackGrp{off, rsrc, g.rows, g.m, g.ntiles, 0, segs[sg].K});
        off += (uint64_t)tile_bytes(bf16, g.rows, g.m) * g.ntiles;
      }
    }
    off = (off + 1023) / 1024 * 1024;
    plan.cta_grp_off[c + 1] = (uint32_t)plan.grps.size();
  }
  if (off / 16 > 0xffffffffull) return "tape too large";
  for (int c = 0; c < ncta; ++c)
    if ((int)cta_grps[c].size() > MAXGRP)
      return "CTA " + std::to_string(c) + " has " + std::to_string(cta_grps[c].size()) + " row groups (> " +
             std::to_string(MAXGRP) + ")";
  plan.tape_bytes = off;
  return "";
}

}  // namespace fq3
