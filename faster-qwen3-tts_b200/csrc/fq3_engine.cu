// fq3_engine.cu -- C ABI implementation (see include/fq3_engine.h): engine lifecycle, weight-tape packing,
// launches of the persistent decode kernel (fq3_decode.cuh).  sm_90a only.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "../../include/fq3_engine.h"
#include "fq3_decode.cuh"
#include "fq3_decode_batch.cuh"

using namespace fq3;

// ------------------------------------------------------------------------------------------------------------
static thread_local char g_err[1024] = "";
static int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
#define CK(call)                                                                                         \
  do {                                                                                                   \
    cudaError_t _e = (call);                                                                             \
    if (_e != cudaSuccess)                                                                               \
      return fail(FQ3_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

// make the engine's device current for the duration of an ABI call and restore the caller's (torch's) device after
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

// host-side record of one request slot (fq3_begin_request latches it; slot_params() hands it to the kernels)
struct SlotHost {
  bool active = false;
  int prefill_len = 0, rope_delta = 0, n_left_pad = 0, max_new = 0, min_new = 0, trailing_len = 0;
  bool text_open = false, text_closed = false;   // fq3_set_text_rows: rows may still follow / the caller closed the text
  int step = 0;   // frames since fq3_begin_request (state[ST_STEP] after the slot's last launch): where its next row goes
  const void* trailing = nullptr;
  const void* tts_pad = nullptr;
  const float* uniforms = nullptr;
  Sampling sp_t{1, 50, 0.9f, 1.0f, 1.05f}, sp_p{1, 50, 0.9f, 1.0f, 1.0f};
};

struct fq3_engine {
  fq3_config cfg;
  bool bf16;
  size_t esz;
  int ncta;
  int dev;
  int max_batch = 1;   // columns a launch may carry
  int max_slots = 1;   // resident request slots (>= max_batch)
  bool loaded = false;
  std::vector<SlotHost> slots;
  size_t pkv_slot = 0;   // bytes of one slot's predictor K (or V) cache
  // paged talker KV cache (kv_row): kv_npages pages of kv_page_bytes; slot s's device page table is kv_tab + s * kv_npt.
  // The host copy of the tables, the owner of every page and the pages a slot maps are what the refusals check.
  void* kv = nullptr;
  int* kv_tab = nullptr;
  int kv_npt = 0, kv_npages = 0;
  size_t kv_page_bytes = 0;
  std::vector<int> kv_tab_host, kv_owner, kv_nmapped;
  int* kv_stage = nullptr;               // pinned: one slot's table on its way to the device
  cudaStream_t kv_stream = nullptr;      // private stream of the table uploads
  // batched decode: activation matrices + per-launch slot table
  float *XB = nullptr, *X1B = nullptr, *QKVB = nullptr, *LOGB = nullptr;
  void *XNB = nullptr, *ATTB = nullptr, *ACTB = nullptr, *PINB = nullptr;
  int* TOKB = nullptr;
  SlotParams* sl_dev = nullptr;
  SlotParams* sl_host = nullptr;  // pinned
  // device buffers (slot-major: slot s starts at s * <per-slot size>)
  void *p_kc = nullptr, *p_vc = nullptr;
  float *X = nullptr, *X1 = nullptr, *QKV = nullptr, *LOGITS = nullptr, *PART = nullptr;
  void *ATT = nullptr, *ACT = nullptr;  // model dtype
  unsigned* bar = nullptr;   // one allocation: grid-barrier and split counters, then X, X1, QKV and LOGITS (xch_bytes)
  size_t xch_bytes = 0;      // cleared before every decode launch
  int* xerr = nullptr;       // sticky exchange-timeout word (KParams::xerr)
  int* xerr_host = nullptr;  // pinned
  int* state = nullptr;
  int* state_host = nullptr;  // pinned
  float* past_hidden = nullptr;
  uint32_t* seen = nullptr;
  float* dbg = nullptr;
  size_t dbg_floats = 0;
  long long dbg_stride = 0;
  int dbg_on = 0;
  uint8_t* tape = nullptr;
  size_t tape_bytes = 0;
  Grp* grps = nullptr;
  uint32_t* segtab = nullptr;
  uint32_t* cta_grp_off = nullptr;
  std::map<std::string, void*> tabs;  // owned small tables (device)
  std::vector<TapeSeg> segs;   // tape_segments(cfg), as of the last load
  int64_t talker_step_bytes = 0, predictor_frame_bytes = 0;
  KParams kp;  // template parameters (static part)
  int64_t launches = 0;
  // K3 prefill: borrowed row-major weights + scratch
  const void *pf_qkv = nullptr, *pf_o = nullptr, *pf_gu = nullptr, *pf_down = nullptr, *pf_head = nullptr;
  void* pf_buf[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  bool pf_ready = false;
};

static size_t smem_bytes() { return sizeof(Smem); }

// ------------------------------------------------------------------------------------------------------------
// small kernels
// ------------------------------------------------------------------------------------------------------------
template <bool BF>
__global__ void set_state_kernel(int* state, float* past_hidden, uint32_t* seen, const void* ph_src, int Ht,
                                 int token, int gen_step) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  if (tid == 0) put_state(state, token, 0, gen_step, FQ3_RUNNING, 0);
  for (int k = tid; k < Ht; k += gridDim.x * blockDim.x) past_hidden[k] = ldw<BF>(ph_src, k);
  for (int k = tid; k < VMAX / 32; k += gridDim.x * blockDim.x) seen[k] = 0u;
}

template <bool BF>
__global__ void get_hidden_kernel(const float* past_hidden, void* dst, int Ht) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < Ht; k += gridDim.x * blockDim.x) stw<BF>(dst, k, past_hidden[k]);
}

// standalone sampler: one CTA of 256 threads running the same sample_block the fused loop uses
template <bool BF>
__global__ void __launch_bounds__(NCT, 1)
    sample_kernel(const __grid_constant__ KParams P, const void* logits, int V, Sampling sp, float u,
                  const long long* hist, int n_hist, int suppress_special, int eos, int suppress_eos,
                  long long* out, float* lp_out) {
  Smem& s = SMEM();
  const int tid = threadIdx.x;
  for (int i = tid; i < VMAX / 32; i += NCT) s.seen[i] = 0u;
  __syncthreads();
  for (int i = tid; i < n_hist; i += NCT) {
    const int v = (int)hist[i];
    if (v >= 0 && v < V) atomicOr(&s.seen[v >> 5], 1u << (v & 31));
  }
  for (int v = tid; v < V; v += NCT) P.LOGITS[v] = ldw<BF>(logits, v);
  __threadfence();
  __syncthreads();
  Ctx c{P, tid, tid >> 5, tid & 31, 0u, 0u};
  const int tok = sample_block<BF>(c, talker_draw(P.LOGITS, V, sp, u, suppress_special != 0, eos, suppress_eos != 0, lp_out));
  if (tid == 0) out[0] = tok;
}

// ------------------------------------------------------------------------------------------------------------
// lifecycle
// ------------------------------------------------------------------------------------------------------------
static int check_stack(const fq3_stack_config& s, const char* nm, int nt) {
  const int qd = s.num_attention_heads * 128, kd = s.num_key_value_heads * 128;
  if (s.hidden_size <= 0 || s.hidden_size % 256 || s.intermediate_size % 256 || qd % 256 || kd % 128)
    return fail(FQ3_ERR_INVALID, "%s: hidden/intermediate/q dims must be multiples of 256 (head_dim fixed at 128)", nm);
  if (s.num_attention_heads % s.num_key_value_heads) return fail(FQ3_ERR_INVALID, "%s: heads %% kv_heads != 0", nm);
  const int mx = std::max(std::max(s.hidden_size, qd), s.intermediate_size);
  if (nt * mx > XS_FLOATS) return fail(FQ3_ERR_INVALID, "%s: %d x max(H,qd,I)=%d exceeds the %d-float staging buffer", nm, nt, mx, XS_FLOATS);
  if (s.vocab_size > VMAX || s.vocab_size % 2) return fail(FQ3_ERR_INVALID, "%s: vocab_size must be even and <= %d", nm, VMAX);
  if (s.num_hidden_layers <= 0) return fail(FQ3_ERR_INVALID, "%s: num_hidden_layers", nm);
  return 0;
}

// bytes of one talker KV page (K and V of KV_PAGE rows of every layer and kv head), pages of max_seq_len rows, and one
// slot's predictor K (or V) cache
static size_t page_bytes(const fq3_config& c, size_t esz) {
  return 2 * kv_half_bytes(c.talker.num_hidden_layers, c.talker.num_key_value_heads, esz);
}
static int pages_per_seq(const fq3_config& c) { return (c.max_seq_len + KV_PAGE - 1) / KV_PAGE; }
static size_t pkv_bytes(const fq3_config& c, size_t esz) {
  return (size_t)c.predictor.num_hidden_layers * c.predictor.num_key_value_heads * 32 * 128 * esz;
}
constexpr size_t STATE_BYTES = 32;   // 8 ints per slot

extern "C" int64_t fq3_slot_bytes(const fq3_config* cfg) {
  if (!cfg) return fail(FQ3_ERR_INVALID, "null argument");
  if (cfg->dtype != FQ3_F32 && cfg->dtype != FQ3_BF16) return fail(FQ3_ERR_INVALID, "dtype must be FQ3_F32 or FQ3_BF16");
  const size_t esz = cfg->dtype == FQ3_BF16 ? 2 : 4;
  return (int64_t)(pages_per_seq(*cfg) * page_bytes(*cfg, esz) + 2 * pkv_bytes(*cfg, esz) + STATE_BYTES +
                   HMAX * sizeof(float) + VMAX / 8);
}

extern "C" int64_t fq3_kv_page_bytes(const fq3_config* cfg) {
  if (!cfg) return fail(FQ3_ERR_INVALID, "null argument");
  if (cfg->dtype != FQ3_F32 && cfg->dtype != FQ3_BF16) return fail(FQ3_ERR_INVALID, "dtype must be FQ3_F32 or FQ3_BF16");
  return (int64_t)page_bytes(*cfg, cfg->dtype == FQ3_BF16 ? 2 : 4);
}

static int engine_alloc(fq3_engine* e, const cudaDeviceProp& prop);

extern "C" int fq3_engine_create(const fq3_config* cfg, fq3_engine** out) {
  if (!cfg || !out) return fail(FQ3_ERR_INVALID, "null argument");
  if (cfg->dtype != FQ3_F32 && cfg->dtype != FQ3_BF16) return fail(FQ3_ERR_INVALID, "dtype must be FQ3_F32 or FQ3_BF16");
  int rc;
  const int max_batch = cfg->max_batch > 0 ? cfg->max_batch : 1;
  const int max_slots = cfg->max_slots != 0 ? cfg->max_slots : max_batch;
  if (max_batch > MAXB) return fail(FQ3_ERR_INVALID, "max_batch %d exceeds %d", cfg->max_batch, MAXB);
  if (max_slots < max_batch) return fail(FQ3_ERR_INVALID, "max_slots %d is smaller than max_batch %d", cfg->max_slots, max_batch);
  if (max_slots > FQ3_MAX_SLOTS) return fail(FQ3_ERR_INVALID, "max_slots %d exceeds %d", cfg->max_slots, FQ3_MAX_SLOTS);
  if ((rc = check_stack(cfg->talker, "talker", 1))) return rc;
  if ((rc = check_stack(cfg->predictor, "predictor", 2))) return rc;
  if (cfg->talker.hidden_size > HMAX) return fail(FQ3_ERR_INVALID, "talker hidden_size > %d", HMAX);
  if (2 * cfg->talker.hidden_size > XS_FLOATS) return fail(FQ3_ERR_INVALID, "talker hidden too large for mtp staging");
  if (cfg->max_seq_len < 8 || cfg->max_seq_len > SEQMAX) return fail(FQ3_ERR_INVALID, "max_seq_len must be in [8,%d]", SEQMAX);
  if (cfg->num_code_groups < 2 || cfg->num_code_groups > 16) return fail(FQ3_ERR_INVALID, "num_code_groups must be in [2,16]");
  if (cfg->rope_positions < cfg->max_seq_len) return fail(FQ3_ERR_INVALID, "rope_positions < max_seq_len");
  if (cfg->kv_pages < 0 || (cfg->kv_pages > 0 && cfg->kv_pages < pages_per_seq(*cfg)))
    return fail(FQ3_ERR_INVALID, "kv_pages %d: a pool must hold one request of max_seq_len=%d rows (%d pages of %d rows)",
                cfg->kv_pages, cfg->max_seq_len, pages_per_seq(*cfg), KV_PAGE);
  int ndev = 0;
  CK(cudaGetDeviceCount(&ndev));
  if (cfg->device < 0 || cfg->device >= ndev) return fail(FQ3_ERR_INVALID, "device %d out of range", cfg->device);
  CK(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9 || prop.minor != 0) return fail(FQ3_ERR_INVALID, "sm_90a required (device is sm_%d%d)", prop.major, prop.minor);
  int coop = 0;
  CK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, cfg->device));
  if (!coop) return fail(FQ3_ERR_INVALID, "device lacks cooperative launch");
  fq3_engine* e = new fq3_engine();
  e->cfg = *cfg;
  e->bf16 = cfg->dtype == FQ3_BF16;
  e->esz = e->bf16 ? 2 : 4;
  e->dev = cfg->device;
  e->ncta = cfg->num_ctas > 0 ? std::min(cfg->num_ctas, prop.multiProcessorCount) : prop.multiProcessorCount;
  e->max_batch = max_batch;
  e->max_slots = max_slots;
  if ((rc = engine_alloc(e, prop))) {
    // the engine owns every pointer it got so far: destroy frees them.  An allocation that did not fit leaves a
    // non-sticky error behind, which must not surface in the caller's next CUDA call
    fq3_engine_destroy(e);
    cudaGetLastError();
    return rc;
  }
  *out = e;
  return 0;
}

// kernel attributes, every device allocation (all of them before the first memset) and the kernel parameter template
static int engine_alloc(fq3_engine* e, const cudaDeviceProp& prop) {
  const fq3_config* cfg = &e->cfg;
  if (e->bf16) {
    CK(cudaFuncSetAttribute(fq3_decode_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
    CK(cudaFuncSetAttribute(fq3_decode_batch_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
    CK(cudaFuncSetAttribute(sample_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
  } else {
    CK(cudaFuncSetAttribute(fq3_decode_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
    CK(cudaFuncSetAttribute(fq3_decode_batch_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
    CK(cudaFuncSetAttribute(sample_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes()));
  }
  int occ = 0;
  if (e->bf16) CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fq3_decode_kernel<true>, NTHREADS, smem_bytes()));
  else CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fq3_decode_kernel<false>, NTHREADS, smem_bytes()));
  if (occ < 1) return fail(FQ3_ERR_INVALID, "decode kernel does not fit on an SM (smem %zu)", smem_bytes());

  const fq3_stack_config &T = cfg->talker, &Pc = cfg->predictor;
  const int MS = e->max_slots;   // per-slot storage; everything a launch needs per column is sized MAXB / MAXCOL below
  e->slots.assign(MS, SlotHost());
  const size_t pkv = pkv_bytes(*cfg, e->esz);
  e->pkv_slot = pkv;
  // talker KV pool: kv_pages = 0 is one max_seq_len run of pages per slot, slot s mapped to its own run for good;
  // a pool of kv_pages > 0 starts with every slot unmapped
  e->kv_npt = pages_per_seq(*cfg);
  e->kv_npages = cfg->kv_pages > 0 ? cfg->kv_pages : MS * e->kv_npt;
  e->kv_page_bytes = page_bytes(*cfg, e->esz);
  e->kv_tab_host.assign((size_t)MS * e->kv_npt, -1);
  e->kv_owner.assign(e->kv_npages, -1);
  e->kv_nmapped.assign(MS, 0);
  if (cfg->kv_pages == 0)
    for (int sl = 0; sl < MS; ++sl) {
      for (int i = 0; i < e->kv_npt; ++i) {
        e->kv_tab_host[(size_t)sl * e->kv_npt + i] = sl * e->kv_npt + i;
        e->kv_owner[sl * e->kv_npt + i] = sl;
      }
      e->kv_nmapped[sl] = e->kv_npt;
    }
  // buffers to clear, once every allocation has succeeded
  std::vector<std::pair<void*, size_t>> zero;
  auto zalloc = [&](void** p, size_t bytes) -> cudaError_t {
    cudaError_t r = cudaMalloc(p, bytes);
    if (r == cudaSuccess) zero.push_back({*p, bytes});
    return r;
  };
  CK(zalloc(&e->kv, e->kv_page_bytes * e->kv_npages));
  CK(cudaMalloc(&e->kv_tab, e->kv_tab_host.size() * sizeof(int)));
  CK(cudaMallocHost(&e->kv_stage, e->kv_npt * sizeof(int)));
  CK(cudaStreamCreateWithFlags(&e->kv_stream, cudaStreamNonBlocking));
  CK(zalloc(&e->p_kc, pkv * MS)); CK(zalloc(&e->p_vc, pkv * MS));
  const int ldX = std::max(T.hidden_size, Pc.hidden_size);
  const int ldQKV = std::max((T.num_attention_heads + 2 * T.num_key_value_heads) * 128,
                             (Pc.num_attention_heads + 2 * Pc.num_key_value_heads) * 128);
  const int ldATT = std::max(T.num_attention_heads, Pc.num_attention_heads) * 128;
  const int ldACT = std::max(T.intermediate_size, Pc.intermediate_size);
  // the barrier words and the four tagged-exchange buffers (fq3_decode.cuh xput) share one allocation, so that the one
  // memset before a launch clears the counters and every exchange tag: tags restart at 1 in each launch
  e->xch_bytes = 32768 + (4 * (size_t)ldX + 2 * (size_t)ldQKV + VMAX) * sizeof(float);
  CK(zalloc((void**)&e->bar, e->xch_bytes));
  e->X = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(e->bar) + 32768);
  e->X1 = e->X + 2 * ldX;
  e->QKV = e->X1 + 2 * ldX;
  e->LOGITS = e->QKV + 2 * ldQKV;
  CK(zalloc((void**)&e->xerr, sizeof(int)));
  CK(cudaMallocHost(&e->xerr_host, sizeof(int)));
  CK(cudaMalloc(&e->ATT, ldATT * e->esz));
  CK(cudaMalloc(&e->ACT, 2 * ldACT * e->esz));
  CK(cudaMalloc(&e->PART, (size_t)T.num_attention_heads * 16 * PART_STRIDE * sizeof(float)));
  CK(zalloc((void**)&e->state, STATE_BYTES * MS));
  CK(cudaMallocHost(&e->state_host, STATE_BYTES * e->max_batch));   // results of one launch: a row per column
  CK(zalloc((void**)&e->past_hidden, (size_t)MS * HMAX * sizeof(float)));
  CK(zalloc((void**)&e->seen, (size_t)MS * (VMAX / 8)));
  if (e->max_batch > 1) {
    // batched decode: activation matrices [column][ld] (column = position in the launch's slot list, predictor pass 0:
    // token * B + column)
    CK(zalloc((void**)&e->XB, (size_t)MAXCOL * ldX * sizeof(float)));
    CK(zalloc((void**)&e->X1B, (size_t)MAXCOL * ldX * sizeof(float)));
    CK(zalloc((void**)&e->QKVB, (size_t)MAXCOL * ldQKV * sizeof(float)));
    CK(zalloc((void**)&e->LOGB, (size_t)MAXB * VMAX * sizeof(float)));
    CK(zalloc(&e->XNB, (size_t)MAXCOL * ldX * e->esz));
    CK(zalloc(&e->ATTB, (size_t)MAXCOL * ldATT * e->esz));
    CK(zalloc(&e->ACTB, (size_t)MAXCOL * ldACT * e->esz));
    CK(zalloc(&e->PINB, (size_t)MAXCOL * HMAX * e->esz));
    CK(zalloc((void**)&e->TOKB, MAXB * sizeof(int)));
    CK(cudaMalloc(&e->sl_dev, MAXB * sizeof(SlotParams)));
    CK(cudaMallocHost(&e->sl_host, MAXB * sizeof(SlotParams)));
  }
  {
    const long long rec_t = 2LL * (T.num_attention_heads + 2 * T.num_key_value_heads) * 128 + 2LL * T.num_attention_heads * 128 + 4LL * T.hidden_size + 2LL * T.intermediate_size;
    const long long rec_p = 2LL * (Pc.num_attention_heads + 2 * Pc.num_key_value_heads) * 128 + 2LL * Pc.num_attention_heads * 128 + 4LL * Pc.hidden_size + 2LL * Pc.intermediate_size;
    e->dbg_stride = std::max(rec_t, rec_p);
    e->dbg_floats = (size_t)e->dbg_stride * std::max(T.num_hidden_layers, Pc.num_hidden_layers);
    CK(zalloc((void**)&e->dbg, e->dbg_floats * sizeof(float)));
  }
  for (auto& z : zero) CK(cudaMemset(z.first, 0, z.second));
  CK(cudaMemcpy(e->kv_tab, e->kv_tab_host.data(), e->kv_tab_host.size() * sizeof(int), cudaMemcpyHostToDevice));
  KParams& k = e->kp;
  memset(&k, 0, sizeof(k));
  auto fill = [&](StackDev& s, const fq3_stack_config& c, int S) {
    s.H = c.hidden_size; s.I = c.intermediate_size; s.L = c.num_hidden_layers;
    s.nH = c.num_attention_heads; s.nKV = c.num_key_value_heads; s.V = c.vocab_size;
    s.qd = s.nH * 128; s.kd = s.nKV * 128; s.rep = s.nH / s.nKV; s.eps = c.rms_norm_eps;
    s.S = S;
  };
  fill(k.t, T, cfg->max_seq_len);
  fill(k.p, Pc, 32);
  k.ncta = e->ncta;
  k.X = e->X; k.X1 = e->X1; k.QKV = e->QKV; k.ATT = e->ATT; k.ACT = e->ACT; k.LOGITS = e->LOGITS;
  k.ldX = ldX; k.ldQKV = ldQKV; k.ldATT = ldATT; k.ldACT = ldACT;
  k.bar = e->bar;
  k.xerr = e->xerr;
  k.XB = e->XB; k.X1B = e->X1B; k.QKVB = e->QKVB; k.LOGB = e->LOGB;
  k.XNB = e->XNB; k.ATTB = e->ATTB; k.ACTB = e->ACTB; k.PINB = e->PINB; k.TOKB = e->TOKB;
  k.nslots = 0; k.sl = e->sl_dev;
  k.has_mtp = cfg->has_mtp_projection; k.ncb = cfg->num_code_groups - 1; k.eos = cfg->codec_eos_token_id;
  k.max_seq_len = cfg->max_seq_len;
  k.dbg = e->dbg; k.dbg_stride_layer = e->dbg_stride;
  {
    // split-key talker attention (bf16 engines): S CTAs per q-head; a slice must fit the 4 ring tiles it may hold
    int Sx = e->bf16 ? std::min(e->ncta / std::max(T.num_attention_heads, 1), 16) : 0;
    if (Sx < 2 || (cfg->max_seq_len + Sx - 1) / Sx > 4 * KVT_KEYS) Sx = 0;
    if (const char* v = getenv("FQ3_ATTN_SPLIT")) Sx = std::min(Sx, std::max(atoi(v), 0)) < 2 ? 0 : std::min(Sx, atoi(v));
    k.attn_split = Sx;
    k.PART = e->PART;
    k.attn_cnt = e->bar + 1024;
  }
  return 0;
}

extern "C" void fq3_engine_destroy(fq3_engine* e) {
  if (!e) return;
  cudaSetDevice(e->dev);
  void* ptrs[] = {e->kv, e->kv_tab, e->p_kc, e->p_vc, e->ATT, e->ACT, e->PART, e->bar, e->xerr,
                  e->state, e->past_hidden, e->seen, e->dbg, e->tape, e->grps, e->segtab, e->cta_grp_off,
                  e->XB, e->X1B, e->QKVB, e->LOGB, e->XNB, e->ATTB, e->ACTB, e->PINB, e->TOKB, e->sl_dev};
  for (void* p : ptrs)
    if (p) cudaFree(p);
  for (auto& kv : e->tabs)
    if (kv.second) cudaFree(kv.second);
  for (void* p : e->pf_buf)
    if (p) cudaFree(p);
  if (e->state_host) cudaFreeHost(e->state_host);
  if (e->xerr_host) cudaFreeHost(e->xerr_host);
  if (e->sl_host) cudaFreeHost(e->sl_host);
  if (e->kv_stage) cudaFreeHost(e->kv_stage);
  if (e->kv_stream) cudaStreamDestroy(e->kv_stream);
  delete e;
}

// table[r][o] = round(bias[o] + sum_k W[o][k] * emb[r][k]) for every row r of the 15 predictor codec embeddings:
// the code predictor's input projection (predictor_graph.py:53 small_to_mtp_projection) of an embedding row depends
// only on the code, so it is tabulated once per weight load instead of being recomputed (GEMV + grid barrier) in 14
// of the 15 passes of every frame.  4 embedding rows per block, one warp per output row.
template <bool BF>
__global__ void mtp_table_kernel(const void* __restrict__ emb, const void* __restrict__ W, const void* __restrict__ bias,
                                 void* __restrict__ table, int K, int N, long long rows) {
  extern __shared__ float es[];  // [4][K]
  const long long r0 = (long long)blockIdx.x * 4;
  for (int i = threadIdx.x; i < 4 * K; i += blockDim.x) {
    const long long r = r0 + i / K;
    es[i] = r < rows ? ldw<BF>(emb, (size_t)r * K + (i % K)) : 0.f;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int o = warp; o < N; o += nw) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int k = lane; k < K; k += 32) {
      const float w = ldw<BF>(W, (size_t)o * K + k);
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] = fmaf(w, es[j * K + k], acc[j]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int s = 16; s; s >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], s);
    if (lane < 4 && r0 + lane < rows) {
      const float b = bias ? ldw<BF>(bias, o) : 0.f;
      const float v = lane == 0 ? acc[0] : (lane == 1 ? acc[1] : (lane == 2 ? acc[2] : acc[3]));
      stw<BF>(table, (size_t)(r0 + lane) * N + o, rnd<BF>(v + b));
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// weights: copy tables, build segments and the per-CTA tape
// ------------------------------------------------------------------------------------------------------------
extern "C" int fq3_engine_load_weights(fq3_engine* e, const fq3_tensor* tensors, int32_t n, void* stream_) {
  if (!e || !tensors) return fail(FQ3_ERR_INVALID, "null argument");
  cudaStream_t stream = (cudaStream_t)stream_;
  DevGuard dev_guard(e->dev);
  std::map<std::string, const fq3_tensor*> tm;
  for (int i = 0; i < n; ++i) tm[tensors[i].name] = &tensors[i];
  const fq3_config& cfg = e->cfg;
  const size_t esz = e->esz;
  auto need = [&](const std::string& nm, int64_t numel, const void** ptr) -> int {
    auto it = tm.find(nm);
    if (it == tm.end()) return fail(FQ3_ERR_INVALID, "missing tensor '%s'", nm.c_str());
    if (it->second->numel != numel)
      return fail(FQ3_ERR_INVALID, "tensor '%s': numel %lld, expected %lld", nm.c_str(), (long long)it->second->numel, (long long)numel);
    *ptr = it->second->dev_ptr;
    return 0;
  };
  int rc;
  // ---- small tables: copied into engine-owned storage
  auto own = [&](const std::string& nm, int64_t numel, size_t elem, const void** devp) -> int {
    const void* src;
    if ((rc = need(nm, numel, &src))) return rc;
    void* dst = nullptr;
    auto it = e->tabs.find(nm);
    if (it != e->tabs.end() && it->second) cudaFree(it->second);
    CK(cudaMalloc(&dst, (size_t)numel * elem));
    CK(cudaMemcpyAsync(dst, src, (size_t)numel * elem, cudaMemcpyDeviceToDevice, stream));
    e->tabs[nm] = dst;
    *devp = dst;
    return 0;
  };
  KParams& k = e->kp;
  struct StackNames { const char* pre; StackDev* s; const fq3_stack_config* c; };
  StackNames sn[2] = {{"t.", &k.t, &cfg.talker}, {"p.", &k.p, &cfg.predictor}};
  for (auto& s : sn) {
    const std::string p = s.pre;
    const int L = s.c->num_hidden_layers, H = s.c->hidden_size;
    if ((rc = own(p + "ln_in", (int64_t)L * H, esz, &s.s->ln_in))) return rc;
    if ((rc = own(p + "ln_post", (int64_t)L * H, esz, &s.s->ln_post))) return rc;
    if ((rc = own(p + "qnorm", (int64_t)L * 128, esz, &s.s->qnorm))) return rc;
    if ((rc = own(p + "knorm", (int64_t)L * 128, esz, &s.s->knorm))) return rc;
    if ((rc = own(p + "ln_f", H, esz, &s.s->ln_f))) return rc;
  }
  {
    const void* p;
    if ((rc = own("t.cos", (int64_t)cfg.rope_positions * 128, 4, &p))) return rc; k.t.cos = (const float*)p;
    if ((rc = own("t.sin", (int64_t)cfg.rope_positions * 128, 4, &p))) return rc; k.t.sin = (const float*)p;
    k.t.npos = cfg.rope_positions;
    if ((rc = own("p.cos", 32 * 128, 4, &p))) return rc; k.p.cos = (const float*)p;
    if ((rc = own("p.sin", 32 * 128, 4, &p))) return rc; k.p.sin = (const float*)p;
    k.p.npos = 32;
    const int Ht = cfg.talker.hidden_size;
    if ((rc = own("t.embed", (int64_t)cfg.talker.vocab_size * Ht, esz, &k.t_embed))) return rc;
    if ((rc = own("p.embeds", (int64_t)k.ncb * cfg.predictor.vocab_size * Ht, esz, &k.p_embeds))) return rc;
    k.mtp_tab = nullptr;
    if (cfg.has_mtp_projection) {
      if ((rc = own("p.mtp_b", cfg.predictor.hidden_size, esz, &k.mtp_b))) return rc;
      // mtp_table_kernel stages 4 embedding rows in shared memory; Ht <= HMAX keeps them within the 48 KB default
      static_assert(4 * HMAX * sizeof(float) <= 48 * 1024, "mtp_table_kernel staging exceeds 48 KB");
      const size_t sm = (size_t)4 * Ht * sizeof(float);
      const void* wm;
      const int Hp = cfg.predictor.hidden_size;
      if ((rc = need("p.mtp_w", (int64_t)Hp * Ht, &wm))) return rc;
      const long long rows = (long long)k.ncb * cfg.predictor.vocab_size;
      void* tab = nullptr;
      auto it = e->tabs.find("p.mtp_table");
      if (it != e->tabs.end() && it->second) cudaFree(it->second);
      CK(cudaMalloc(&tab, (size_t)rows * Hp * esz));
      e->tabs["p.mtp_table"] = tab;
      const unsigned nb = (unsigned)((rows + 3) / 4);
      if (e->bf16) mtp_table_kernel<true><<<nb, 256, sm, stream>>>(k.p_embeds, wm, k.mtp_b, tab, Ht, Hp, rows);
      else mtp_table_kernel<false><<<nb, 256, sm, stream>>>(k.p_embeds, wm, k.mtp_b, tab, Ht, Hp, rows);
      CK(cudaGetLastError());
      k.mtp_tab = tab;
    } else {
      k.mtp_b = nullptr;
    }
  }
  // ---- segments: their tensors resolved by name into the row-source table, then planned over the CTAs
  TapeSegments T = tape_segments(cfg);
  std::vector<const void*> rowsrc;
  for (const TapeSeg& s : T.segs) {
    const void* w[3];
    for (size_t i = 0; i < s.runs.size(); ++i)
      if ((rc = need(s.runs[i].tensor, s.runs[i].tensor_rows * s.K, &w[i]))) return rc;
    tape_rows(s, w, esz, rowsrc);
  }
  TapePlan plan;
  const std::string err = plan_tape(T.segs, e->ncta, e->bf16, plan);
  if (!err.empty()) return fail(FQ3_ERR_INVALID, "%s", err.c_str());
  k.t.seg_base = T.seg_base[0]; k.t.seg_head = T.seg_head[0];
  k.p.seg_base = T.seg_base[1]; k.p.seg_head = T.seg_head[1];
  k.seg_mtp = T.seg_mtp;
  k.nseg = (int)T.segs.size();
  e->segs = std::move(T.segs);
  // ---- upload tables, pack.  A reload frees what the previous load allocated.
  auto upload = [&](auto** dst, const auto& v) -> int {
    if (*dst) cudaFree((void*)*dst);
    *dst = nullptr;
    CK(cudaMalloc(dst, v.size() * sizeof(v[0])));
    CK(cudaMemcpyAsync((void*)*dst, v.data(), v.size() * sizeof(v[0]), cudaMemcpyHostToDevice, stream));
    return 0;
  };
  if (e->tape) { cudaFree(e->tape); e->tape = nullptr; }
  CK(cudaMalloc(&e->tape, plan.tape_bytes));
  e->tape_bytes = plan.tape_bytes;
  const void** d_rowsrc = nullptr;
  PackGrp* d_pack = nullptr;
  if ((rc = upload(&e->grps, plan.grps)) || (rc = upload(&e->segtab, plan.segtab)) ||
      (rc = upload(&e->cta_grp_off, plan.cta_grp_off)) || (rc = upload(&d_rowsrc, rowsrc)) ||
      (rc = upload(&d_pack, plan.pack)))
    return rc;
  const int npack = (int)plan.pack.size(), grid = std::min(npack, 132 * 16);
  if (e->bf16) pack_mma_kernel<<<grid, 256, 0, stream>>>(d_pack, npack, d_rowsrc, e->tape);
  else pack_kernel<<<grid, 256, 0, stream>>>(d_pack, npack, d_rowsrc, e->tape);
  e->launches++;
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(stream));
  cudaFree(d_rowsrc);
  cudaFree(d_pack);
  k.tape = e->tape; k.grps = e->grps; k.segtab = e->segtab; k.cta_grp_off = e->cta_grp_off;
  // ---- byte accounting (algorithmic bytes): a stack's layers, its heads and the MTP projection are consecutive segments
  auto bytes = [&](int sg0, int n) {
    uint64_t b = 0;
    for (int sg = sg0; sg < sg0 + n; ++sg) b += (uint64_t)e->segs[sg].rows * e->segs[sg].K * esz;
    return b;
  };
  e->talker_step_bytes = (int64_t)bytes(k.t.seg_base, 4 * k.t.L + 1);
  e->predictor_frame_bytes = (int64_t)(k.ncb * bytes(k.p.seg_base, 4 * k.p.L) + bytes(k.p.seg_head, k.ncb + (k.seg_mtp >= 0)));
  e->loaded = true;
  return 0;
}

// ------------------------------------------------------------------------------------------------------------
// launches
// ------------------------------------------------------------------------------------------------------------
// one cooperative launch of a persistent decode kernel: the single-sequence kernel (kp.nslots == 0) or the batched
// one, in the engine's dtype, with the grid-barrier and attention-split counters and the exchange tags cleared first
static int launch_decode(fq3_engine* e, const KParams& kp, cudaStream_t stream) {
  const void* fn = kp.nslots == 0 ? (e->bf16 ? (const void*)fq3_decode_kernel<true> : (const void*)fq3_decode_kernel<false>)
                                  : (e->bf16 ? (const void*)fq3_decode_batch_kernel<true> : (const void*)fq3_decode_batch_kernel<false>);
  CK(cudaMemsetAsync(e->bar, 0, e->xch_bytes, stream));
  void* args[] = {(void*)&kp};
  CK(cudaLaunchCooperativeKernel(fn, dim3(e->ncta), dim3(NTHREADS), args, smem_bytes(), stream));
  e->launches++;
  return 0;
}

static Sampling to_sampling(const fq3_sampling* s) {
  Sampling r;
  r.do_sample = s->do_sample; r.top_k = s->top_k; r.temperature = s->temperature; r.top_p = s->top_p;
  r.penalty = s->repetition_penalty;
  return r;
}

// the bound on slot ids by the name the engine's creator gave it: an engine created without max_slots has one number,
// max_batch, and callers written for it read (and match) messages that name it
static const char* slot_bound(const fq3_engine* e) { return e->max_slots == e->max_batch ? "max_batch" : "max_slots"; }
static int check_slot(fq3_engine* e, int slot) {
  if (slot < 0 || slot >= e->max_slots)
    return fail(FQ3_ERR_INVALID, "slot %d outside [0, %s=%d)", slot, slot_bound(e), e->max_slots);
  return 0;
}
// cache rows slot s has pages for; the refusals below keep every kernel inside them
static int kv_rows(const fq3_engine* e, int s) { return e->kv_nmapped[s] * KV_PAGE; }
static int check_rows(fq3_engine* e, int slot, long long rows, const char* what) {
  if (rows > kv_rows(e, slot))
    return fail(FQ3_ERR_INVALID, "slot %d: %s needs cache rows [0, %lld) but its pages map %d rows", slot, what, rows,
                kv_rows(e, slot));
  return 0;
}
static void* slot_pk(fq3_engine* e, int s) { return (uint8_t*)e->p_kc + (size_t)s * e->pkv_slot; }
static void* slot_pv(fq3_engine* e, int s) { return (uint8_t*)e->p_vc + (size_t)s * e->pkv_slot; }

// the kernels' record of slot s: its caches and state, the request it latched, where its codes go
static SlotParams slot_params(fq3_engine* e, int s, int n_frames, long long* codes_out, float* logprob_out) {
  const SlotHost& h = e->slots[s];
  SlotParams p;
  p.kv = e->kv; p.kv_pages = e->kv_tab + (size_t)s * e->kv_npt; p.pkc = slot_pk(e, s); p.pvc = slot_pv(e, s);
  p.state = e->state + 8 * s;
  p.past_hidden = e->past_hidden + (size_t)s * HMAX;
  p.seen = e->seen + (size_t)s * (VMAX / 32);
  p.trailing = h.trailing; p.tts_pad = h.tts_pad; p.uniforms = h.uniforms;
  p.codes_out = codes_out;
  p.logprob_out = logprob_out;
  p.prefill_len = h.prefill_len; p.rope_delta = h.rope_delta; p.n_left_pad = h.n_left_pad;
  p.max_new = h.max_new; p.min_new = h.min_new; p.trailing_len = h.trailing_len;
  p.text_open = h.text_open ? 1 : 0;
  p.n_frames = n_frames;
  p.sp_t = h.sp_t; p.sp_p = h.sp_p;
  return p;
}

// kernel parameters of a step-wise single-sequence launch on slot s
static KParams kp_for_slot(fq3_engine* e, int s, long long* codes_out) {
  KParams kp = e->kp;
  kp.req = slot_params(e, s, 0, codes_out, nullptr);
  kp.nslots = 0;
  return kp;
}

// rows [0,P) of one layer between the caller's k,v [n_kv, P, 128] and the slot's pages: per page, one 2-D copy of the
// page's rows of every kv head (they are KV_PAGE rows apart in the page, P rows apart in the caller's tensor)
static int copy_kv(fq3_engine* e, int slot, int layer, void* k, void* v, int P, bool to_cache, cudaStream_t stream) {
  const int L = e->cfg.talker.num_hidden_layers, nKV = e->cfg.talker.num_key_value_heads;
  const int* pages = e->kv_tab_host.data() + (size_t)slot * e->kv_npt;
  const size_t rowb = 128 * e->esz, pitch = (size_t)P * rowb;
  for (int t0 = 0; t0 < P; t0 += KV_PAGE) {
    const size_t w = (size_t)std::min(KV_PAGE, P - t0) * rowb;
    for (int which = 0; which < 2; ++which) {
      uint8_t* c = kv_row(e->kv, L, nKV, e->esz, pages, which, layer, 0, t0);
      const size_t cp = kv_row(e->kv, L, nKV, e->esz, pages, which, layer, 1, t0) - c;   // kv head to kv head
      uint8_t* u = (uint8_t*)(which ? v : k) + (size_t)t0 * rowb;
      if (to_cache) CK(cudaMemcpy2DAsync(c, cp, u, pitch, w, nKV, cudaMemcpyDeviceToDevice, stream));
      else CK(cudaMemcpy2DAsync(u, pitch, c, cp, w, nKV, cudaMemcpyDeviceToDevice, stream));
    }
  }
  return 0;
}

extern "C" int fq3_import_kv(fq3_engine* e, int32_t slot, int32_t layer, const void* k_dev, const void* v_dev, int32_t P,
                             void* stream_) {
  if (!e || !k_dev || !v_dev) return fail(FQ3_ERR_INVALID, "null argument");
  int rc;
  if ((rc = check_slot(e, slot))) return rc;
  if (P > e->cfg.max_seq_len)
    return fail(FQ3_ERR_TOO_LONG, "Input is too long: prefill has %d tokens but max_seq_len=%d. Use shorter text or shorter reference audio.", P, e->cfg.max_seq_len);
  if (layer < 0 || layer >= e->cfg.talker.num_hidden_layers) return fail(FQ3_ERR_INVALID, "layer out of range");
  if ((rc = check_rows(e, slot, P, "fq3_import_kv"))) return rc;
  DevGuard dev_guard(e->dev);
  return copy_kv(e, slot, layer, (void*)k_dev, (void*)v_dev, P, true, (cudaStream_t)stream_);
}

extern "C" int fq3_export_kv(fq3_engine* e, int32_t slot, int32_t layer, void* k_dev, void* v_dev, int32_t P, void* stream_) {
  if (!e || !k_dev || !v_dev) return fail(FQ3_ERR_INVALID, "null argument");
  int rc;
  if ((rc = check_slot(e, slot))) return rc;
  if (P < 0 || P > e->cfg.max_seq_len) return fail(FQ3_ERR_INVALID, "P outside the cache");
  if (layer < 0 || layer >= e->cfg.talker.num_hidden_layers) return fail(FQ3_ERR_INVALID, "layer out of range");
  if ((rc = check_rows(e, slot, P, "fq3_export_kv"))) return rc;
  DevGuard dev_guard(e->dev);
  return copy_kv(e, slot, layer, k_dev, v_dev, P, false, (cudaStream_t)stream_);
}

extern "C" int fq3_set_generation_state(fq3_engine* e, int32_t slot, int32_t n_left_pad, int32_t rope_delta) {
  if (!e) return fail(FQ3_ERR_INVALID, "null argument");
  int rc;
  if ((rc = check_slot(e, slot))) return rc;
  e->slots[slot].n_left_pad = n_left_pad;
  e->slots[slot].rope_delta = rope_delta;
  return 0;
}

extern "C" int fq3_talker_step(fq3_engine* e, int32_t slot, const void* embeds_dev, int32_t position, void* hidden_out_dev,
                               void* stream_) {
  if (!e || !embeds_dev || !hidden_out_dev) return fail(FQ3_ERR_INVALID, "null argument");
  if (!e->loaded) return fail(FQ3_ERR_STATE, "weights not loaded");
  int rc;
  if ((rc = check_slot(e, slot))) return rc;
  if (position < 0 || position >= e->cfg.max_seq_len) return fail(FQ3_ERR_INVALID, "position %d outside the cache", position);
  if ((rc = check_rows(e, slot, (long long)position + 1, "fq3_talker_step"))) return rc;
  DevGuard dev_guard(e->dev);
  KParams kp = kp_for_slot(e, slot, nullptr);
  kp.mode = MODE_TALKER_STEP;
  kp.in_embeds = embeds_dev; kp.hidden_out = hidden_out_dev; kp.position = position;
  kp.dbg_on = e->dbg_on;
  return launch_decode(e, kp, (cudaStream_t)stream_);
}

extern "C" int fq3_predictor_run(fq3_engine* e, int32_t slot, const void* pred_input_dev, const fq3_sampling* sp,
                                 const float* uniforms_dev, int64_t* codes_out_dev, void* stream_) {
  if (!e || !pred_input_dev || !sp || !codes_out_dev) return fail(FQ3_ERR_INVALID, "null argument");
  if (!e->loaded) return fail(FQ3_ERR_STATE, "weights not loaded");
  int rc;
  if ((rc = check_slot(e, slot))) return rc;
  if (sp->do_sample && !uniforms_dev) return fail(FQ3_ERR_INVALID, "do_sample needs uniforms");
  DevGuard dev_guard(e->dev);
  KParams kp = kp_for_slot(e, slot, (long long*)codes_out_dev);
  kp.mode = MODE_PRED_RUN;
  kp.pred_input = pred_input_dev; kp.pred_uniforms = uniforms_dev;
  kp.req.sp_p = to_sampling(sp);
  kp.dbg_on = e->dbg_on;
  return launch_decode(e, kp, (cudaStream_t)stream_);
}

extern "C" int fq3_sample_logits_lp(fq3_engine* e, const void* logits_dev, int32_t V, const fq3_sampling* sp, float u,
                                    const int64_t* history_dev, int32_t n_hist, int32_t suppress_special, int32_t eos_id,
                                    int32_t suppress_eos, int64_t* token_out_dev, float* logprob_out_dev, void* stream_) {
  if (!e || !logits_dev || !sp || !token_out_dev) return fail(FQ3_ERR_INVALID, "null argument");
  if (V <= 0 || V > VMAX) return fail(FQ3_ERR_INVALID, "V out of range");
  DevGuard dev_guard(e->dev);
  cudaStream_t stream = (cudaStream_t)stream_;
  const Sampling s = to_sampling(sp);
  if (e->bf16)
    sample_kernel<true><<<1, NCT, smem_bytes(), stream>>>(e->kp, logits_dev, V, s, u, (const long long*)history_dev, history_dev ? n_hist : 0, suppress_special, eos_id, suppress_eos, (long long*)token_out_dev, logprob_out_dev);
  else
    sample_kernel<false><<<1, NCT, smem_bytes(), stream>>>(e->kp, logits_dev, V, s, u, (const long long*)history_dev, history_dev ? n_hist : 0, suppress_special, eos_id, suppress_eos, (long long*)token_out_dev, logprob_out_dev);
  e->launches++;
  CK(cudaGetLastError());
  return 0;
}

extern "C" int fq3_sample_logits(fq3_engine* e, const void* logits_dev, int32_t V, const fq3_sampling* sp, float u,
                                 const int64_t* history_dev, int32_t n_hist, int32_t suppress_special, int32_t eos_id,
                                 int32_t suppress_eos, int64_t* token_out_dev, void* stream) {
  return fq3_sample_logits_lp(e, logits_dev, V, sp, u, history_dev, n_hist, suppress_special, eos_id, suppress_eos,
                              token_out_dev, nullptr, stream);
}

extern "C" int fq3_begin_request(fq3_engine* e, int32_t slot, const fq3_request* rq, const void* past_hidden_dev,
                                 const void* trailing_text_dev, const void* tts_pad_dev, const float* uniforms_dev,
                                 const fq3_sampling* sp_talker, const fq3_sampling* sp_predictor, void* stream_) {
  if (!e || !rq || !past_hidden_dev || !tts_pad_dev || !sp_talker || !sp_predictor) return fail(FQ3_ERR_INVALID, "null argument");
  if (!e->loaded) return fail(FQ3_ERR_STATE, "weights not loaded");
  int rc;
  if ((rc = check_slot(e, slot))) return rc;
  if (rq->prefill_len > e->cfg.max_seq_len)
    return fail(FQ3_ERR_TOO_LONG, "Input is too long: prefill has %d tokens but max_seq_len=%d. Use shorter text or shorter reference audio.", rq->prefill_len, e->cfg.max_seq_len);
  if ((sp_talker->do_sample || sp_predictor->do_sample) && !uniforms_dev) return fail(FQ3_ERR_INVALID, "sampling needs uniforms");
  if (rq->trailing_len > 0 && !trailing_text_dev) return fail(FQ3_ERR_INVALID, "trailing_len > 0 but no trailing text");
  if (rq->first_token < 0 || rq->first_token >= e->cfg.talker.vocab_size) return fail(FQ3_ERR_INVALID, "first_token out of range");
  DevGuard dev_guard(e->dev);
  cudaStream_t stream = (cudaStream_t)stream_;
  SlotHost& h = e->slots[slot];
  h.prefill_len = rq->prefill_len; h.rope_delta = rq->rope_delta; h.n_left_pad = rq->n_left_pad;
  h.max_new = rq->max_new_tokens; h.min_new = rq->min_new_tokens; h.trailing_len = rq->trailing_len;
  h.trailing = trailing_text_dev; h.tts_pad = tts_pad_dev; h.uniforms = uniforms_dev;
  h.text_open = false; h.text_closed = false;
  h.step = 0;
  h.sp_t = to_sampling(sp_talker); h.sp_p = to_sampling(sp_predictor);
  int* st = e->state + 8 * slot;
  float* ph = e->past_hidden + (size_t)slot * HMAX;
  uint32_t* seen = e->seen + (size_t)slot * (VMAX / 32);
  if (e->bf16) set_state_kernel<true><<<4, 256, 0, stream>>>(st, ph, seen, past_hidden_dev, e->cfg.talker.hidden_size, rq->first_token, rq->gen_step);
  else set_state_kernel<false><<<4, 256, 0, stream>>>(st, ph, seen, past_hidden_dev, e->cfg.talker.hidden_size, rq->first_token, rq->gen_step);
  e->launches++;
  CK(cudaGetLastError());
  h.active = true;
  return 0;
}

extern "C" int fq3_set_text_rows(fq3_engine* e, int32_t slot, int32_t trailing_len, int32_t open) {
  if (!e) return fail(FQ3_ERR_INVALID, "null argument");
  int rc;
  if ((rc = check_slot(e, slot))) return rc;
  SlotHost& h = e->slots[slot];
  if (!h.active) return fail(FQ3_ERR_STATE, "fq3_begin_request has not been called for slot %d", slot);
  if (trailing_len < h.trailing_len)
    return fail(FQ3_ERR_INVALID, "slot %d: trailing_len %d < %d (rows already announced cannot be withdrawn)", slot, trailing_len, h.trailing_len);
  if (open && h.text_closed) return fail(FQ3_ERR_STATE, "slot %d: the text was closed and cannot be reopened", slot);
  // a closed slot may already have fed tts_pad past its last row: a row announced now would follow the end of the text
  if (h.text_closed && trailing_len != h.trailing_len)
    return fail(FQ3_ERR_STATE, "slot %d: the text was closed at %d rows; trailing_len cannot grow to %d", slot, h.trailing_len, trailing_len);
  if (trailing_len > 0 && !h.trailing) return fail(FQ3_ERR_INVALID, "slot %d: trailing_len > 0 but fq3_begin_request latched no trailing text", slot);
  h.trailing_len = trailing_len;
  h.text_open = open != 0;
  h.text_closed = open == 0;
  return 0;
}

// fused launch of slots[0..n): column j emits up to n_frames[j] frames into row j of the [n][max_frames][16] outputs.
// One slot runs on the single-sequence kernel, more become the columns of one batched pass over the weight tape.
static int launch_fused(fq3_engine* e, const int32_t* slots, int n, const int32_t* n_frames, int max_frames,
                        long long* codes_out_dev, float* logprob_out_dev, cudaStream_t stream) {
  KParams kp = e->kp;
  kp.mode = MODE_FUSED;
  kp.n_frames = max_frames;   // the producer warp's bound: no slot runs longer
  kp.dbg_on = e->dbg_on & 2;  // timing probes only; layer dumps belong to the step-wise entry points
  if (n == 1) {
    kp.req = slot_params(e, slots[0], n_frames[0], codes_out_dev, logprob_out_dev);
    kp.nslots = 0;
  } else {
    if (!e->sl_dev) return fail(FQ3_ERR_STATE, "engine was created with max_batch = 1");
    if (n > e->ncta) return fail(FQ3_ERR_INVALID, "%d slots need at least as many CTAs (engine has %d)", n, e->ncta);
    for (int j = 0; j < n; ++j)
      e->sl_host[j] = slot_params(e, slots[j], n_frames[j], codes_out_dev + (size_t)j * max_frames * 16,
                                  logprob_out_dev ? logprob_out_dev + (size_t)j * max_frames * 16 : nullptr);
    CK(cudaMemcpyAsync(e->sl_dev, e->sl_host, (size_t)n * sizeof(SlotParams), cudaMemcpyHostToDevice, stream));
    kp.nslots = n;
    kp.sl = e->sl_dev;
  }
  return launch_decode(e, kp, stream);
}

// numerics probe: ONE batched GEMV (the kernel the batched decode path is built from) over a weight segment
extern "C" int fq3_debug_gemv(fq3_engine* e, int32_t stack, int32_t layer, int32_t which, int32_t ncols, const void* x_dev,
                              void* out_dev, void* stream_) {
  if (!e || !x_dev || !out_dev) return fail(FQ3_ERR_INVALID, "null argument");
  if (!e->loaded) return fail(FQ3_ERR_STATE, "weights not loaded");
  if (!e->sl_dev) return fail(FQ3_ERR_STATE, "engine was created with max_batch = 1");
  if (ncols < 1 || ncols > MAXCOL) return fail(FQ3_ERR_INVALID, "ncols out of range");
  const StackDev& S = stack == 0 ? e->kp.t : e->kp.p;
  int sg;
  if (which >= 0 && which < 4) {
    if (layer < 0 || layer >= S.L) return fail(FQ3_ERR_INVALID, "layer out of range");
    sg = S.seg_base + 4 * layer + which;
  } else if (which == 4) {
    sg = S.seg_head + (stack == 0 ? 0 : layer);
  } else {
    return fail(FQ3_ERR_INVALID, "which must be 0..4 (qkv, o, gate/up, down, head)");
  }
  DevGuard dev_guard(e->dev);
  KParams kp = e->kp;
  kp.mode = MODE_GEMV_TEST;
  kp.nslots = 1;
  kp.sl = e->sl_dev;
  kp.n_frames = 0;
  kp.dbg_on = 0;
  kp.gt_seg = sg; kp.gt_K = e->segs[sg].K; kp.gt_rows = e->segs[sg].rows; kp.gt_ncols = ncols;
  kp.gt_swiglu = which == 2 ? 1 : 0;
  kp.gt_x = x_dev; kp.gt_out = out_dev;
  return launch_decode(e, kp, (cudaStream_t)stream_);
}

extern "C" int fq3_decode_chunk_n(fq3_engine* e, const int32_t* slots, int32_t n_slots, const int32_t* n_frames,
                                  int64_t* codes_out_dev, float* logprob_out_dev, fq3_chunk_result* res, void* stream_) {
  if (!e || !slots || !n_frames || !codes_out_dev || !res) return fail(FQ3_ERR_INVALID, "null argument");
  if (n_slots <= 0 || n_slots > e->max_batch)
    return fail(FQ3_ERR_INVALID, "n_slots %d outside [1, max_batch=%d] (columns of one launch; the engine holds %d slots)",
                n_slots, e->max_batch, e->max_slots);
  int rc, max_frames = 0;
  for (int j = 0; j < n_slots; ++j) {
    if (n_frames[j] <= 0) return fail(FQ3_ERR_INVALID, "n_frames must be positive (slot %d: %d)", slots[j], n_frames[j]);
    max_frames = std::max(max_frames, (int)n_frames[j]);
    if ((rc = check_slot(e, slots[j]))) return rc;
    if (!e->slots[slots[j]].active) return fail(FQ3_ERR_STATE, "fq3_begin_request has not been called for slot %d", slots[j]);
    for (int i = 0; i < j; ++i)
      if (slots[i] == slots[j]) return fail(FQ3_ERR_INVALID, "slot %d listed twice", slots[j]);
    // frame s writes cache row prefill_len + s unless that row is the last one (the max_seq_len rule)
    const SlotHost& h = e->slots[slots[j]];
    const long long rows = std::min((long long)h.prefill_len + h.step + n_frames[j], (long long)e->cfg.max_seq_len - 1);
    if ((rc = check_rows(e, slots[j], rows, "a frame budget"))) return rc;
  }
  DevGuard dev_guard(e->dev);
  cudaStream_t stream = (cudaStream_t)stream_;
  if ((rc = launch_fused(e, slots, n_slots, n_frames, max_frames, (long long*)codes_out_dev, logprob_out_dev, stream))) return rc;
  for (int j = 0; j < n_slots; ++j)
    CK(cudaMemcpyAsync(e->state_host + 8 * j, e->state + 8 * slots[j], 32, cudaMemcpyDeviceToHost, stream));
  CK(cudaMemcpyAsync(e->xerr_host, e->xerr, sizeof(int), cudaMemcpyDeviceToHost, stream));
  CK(cudaStreamSynchronize(stream));
  // a tagged exchange gave up waiting in this launch or an earlier one (a protocol error, never expected): the
  // activations of that launch are undefined, and so is every result since
  if (*e->xerr_host) return fail(FQ3_ERR_CUDA, "decode kernel: an activation exchange timed out; results are undefined");
  for (int j = 0; j < n_slots; ++j) {
    const int* st = e->state_host + 8 * j;
    res[j].next_token = st[ST_TOKEN];
    res[j].total_frames = st[ST_STEP];
    res[j].finished = st[ST_FIN];
    res[j].frames_emitted = st[ST_EMIT];
    e->slots[slots[j]].step = st[ST_STEP];
  }
  return 0;
}

extern "C" int fq3_decode_chunk_lp(fq3_engine* e, const int32_t* slots, int32_t n_slots, int32_t n_frames,
                                   int64_t* codes_out_dev, float* logprob_out_dev, fq3_chunk_result* res, void* stream) {
  int32_t budgets[MAXB];
  for (int j = 0; j < MAXB; ++j) budgets[j] = n_frames;
  return fq3_decode_chunk_n(e, slots, n_slots, budgets, codes_out_dev, logprob_out_dev, res, stream);
}

extern "C" int fq3_decode_chunk(fq3_engine* e, const int32_t* slots, int32_t n_slots, int32_t n_frames,
                                int64_t* codes_out_dev, fq3_chunk_result* res, void* stream) {
  return fq3_decode_chunk_lp(e, slots, n_slots, n_frames, codes_out_dev, nullptr, res, stream);
}

extern "C" int fq3_get_past_hidden(fq3_engine* e, int32_t slot, void* dst_dev, void* stream_) {
  if (!e || !dst_dev) return fail(FQ3_ERR_INVALID, "null argument");
  int rc;
  if ((rc = check_slot(e, slot))) return rc;
  DevGuard dev_guard(e->dev);
  cudaStream_t stream = (cudaStream_t)stream_;
  const float* ph = e->past_hidden + (size_t)slot * HMAX;
  if (e->bf16) get_hidden_kernel<true><<<4, 256, 0, stream>>>(ph, dst_dev, e->cfg.talker.hidden_size);
  else get_hidden_kernel<false><<<4, 256, 0, stream>>>(ph, dst_dev, e->cfg.talker.hidden_size);
  e->launches++;
  CK(cudaGetLastError());
  return 0;
}

extern "C" int fq3_debug_enable(fq3_engine* e, int32_t on) {
  if (!e) return fail(FQ3_ERR_INVALID, "null argument");
  e->dbg_on = on;
  return 0;
}

extern "C" int fq3_debug_read(fq3_engine* e, int64_t offset, int64_t count, float* host_dst) {
  if (!e || !host_dst) return fail(FQ3_ERR_INVALID, "null argument");
  if (offset < 0 || count < 0 || (size_t)(offset + count) > e->dbg_floats) return fail(FQ3_ERR_INVALID, "debug range outside the buffer (%zu floats)", e->dbg_floats);
  DevGuard dev_guard(e->dev);
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(host_dst, e->dbg + offset, (size_t)count * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}

extern "C" int fq3_tape_bytes(fq3_engine* e, int64_t* talker_step_bytes, int64_t* predictor_frame_bytes) {
  if (!e) return fail(FQ3_ERR_INVALID, "null argument");
  if (talker_step_bytes) *talker_step_bytes = e->talker_step_bytes;
  if (predictor_frame_bytes) *predictor_frame_bytes = e->predictor_frame_bytes;
  return 0;
}

// ---- paged talker KV cache
extern "C" int fq3_map_kv_pages(fq3_engine* e, int32_t slot, const int32_t* pages, int32_t n) {
  if (!e || (n > 0 && !pages)) return fail(FQ3_ERR_INVALID, "null argument");
  int rc;
  if ((rc = check_slot(e, slot))) return rc;
  if (n < 0 || n > e->kv_npt)
    return fail(FQ3_ERR_INVALID, "slot %d: %d pages outside [0, %d] (max_seq_len=%d rows)", slot, n, e->kv_npt, e->cfg.max_seq_len);
  for (int i = 0; i < n; ++i) {
    if (pages[i] < 0 || pages[i] >= e->kv_npages)
      return fail(FQ3_ERR_INVALID, "slot %d: page %d outside [0, %d)", slot, pages[i], e->kv_npages);
    for (int j = 0; j < i; ++j)
      if (pages[j] == pages[i]) return fail(FQ3_ERR_INVALID, "slot %d: page %d listed twice", slot, pages[i]);
    const int o = e->kv_owner[pages[i]];
    if (o >= 0 && o != slot) return fail(FQ3_ERR_INVALID, "slot %d: page %d is mapped to slot %d", slot, pages[i], o);
  }
  DevGuard dev_guard(e->dev);
  int* tab = e->kv_tab_host.data() + (size_t)slot * e->kv_npt;
  for (int i = 0; i < e->kv_npt; ++i) {
    if (tab[i] >= 0) e->kv_owner[tab[i]] = -1;
    tab[i] = i < n ? pages[i] : -1;
  }
  for (int i = 0; i < n; ++i) e->kv_owner[pages[i]] = slot;
  e->kv_nmapped[slot] = n;
  memcpy(e->kv_stage, tab, e->kv_npt * sizeof(int));
  CK(cudaMemcpyAsync(e->kv_tab + (size_t)slot * e->kv_npt, e->kv_stage, e->kv_npt * sizeof(int), cudaMemcpyHostToDevice,
                     e->kv_stream));
  CK(cudaStreamSynchronize(e->kv_stream));
  return 0;
}

extern "C" int fq3_slot_kv_rows(fq3_engine* e, int32_t slot) {
  if (!e) return fail(FQ3_ERR_INVALID, "null argument");
  int rc;
  if ((rc = check_slot(e, slot))) return rc;
  return kv_rows(e, slot);
}

extern "C" int fq3_kv_pool_pages(fq3_engine* e) { return e ? e->kv_npages : 0; }

static int copy_pages(fq3_engine* e, const int32_t* pages, int32_t n, void* mem, bool out, void* stream_) {
  if (!e || (n > 0 && (!pages || !mem))) return fail(FQ3_ERR_INVALID, "null argument");
  if (n < 0) return fail(FQ3_ERR_INVALID, "n %d < 0", n);
  for (int i = 0; i < n; ++i) {
    if (pages[i] < 0 || pages[i] >= e->kv_npages) return fail(FQ3_ERR_INVALID, "page %d outside [0, %d)", pages[i], e->kv_npages);
    for (int j = 0; j < i; ++j)
      if (pages[j] == pages[i]) return fail(FQ3_ERR_INVALID, "page %d listed twice", pages[i]);
  }
  DevGuard dev_guard(e->dev);
  const int L = e->cfg.talker.num_hidden_layers, nKV = e->cfg.talker.num_key_value_heads;
  for (int i = 0; i < n; ++i) {
    uint8_t* pg = kv_row(e->kv, L, nKV, e->esz, &pages[i], 0, 0, 0, 0);   // a page is one block: its first row
    uint8_t* m = (uint8_t*)mem + (size_t)i * e->kv_page_bytes;
    CK(cudaMemcpyAsync(out ? m : pg, out ? pg : m, e->kv_page_bytes, cudaMemcpyDefault, (cudaStream_t)stream_));
  }
  return 0;
}
extern "C" int fq3_kv_pages_to(fq3_engine* e, const int32_t* pages, int32_t n, void* dst, void* stream) {
  return copy_pages(e, pages, n, dst, true, stream);
}
extern "C" int fq3_kv_pages_from(fq3_engine* e, const int32_t* pages, int32_t n, const void* src, void* stream) {
  return copy_pages(e, pages, n, (void*)src, false, stream);
}

extern "C" int fq3_num_ctas(fq3_engine* e) { return e ? e->ncta : 0; }
extern "C" int64_t fq3_launch_count(fq3_engine* e) { return e ? e->launches : 0; }
extern "C" const char* fq3_last_error(void) { return g_err; }
extern "C" int fq3_max_batch(fq3_engine* e) { return e ? e->max_batch : 0; }
extern "C" int fq3_max_slots(fq3_engine* e) { return e ? e->max_slots : 0; }
extern "C" const char* fq3_version(void) { return "fq3-h100 0.3.0 (sm_90a)"; }

#include "fq3_prefill.cuh"

// numerics probe: ONE launch of the dense-layer GEMM of K3 / K4 with the caller's arguments, unchanged.  Refused here:
// only what would make the kernel divide by zero or dereference a missing parameter array, and operands the SwiGLU
// epilogue would silently ignore.  Every shape and alignment rule is the kernel's own (fq3gemm::gemm refuses before it
// launches anything).
extern "C" int fq3_debug_conv_gemm(const fq3_conv_probe* p, void* stream) {
  if (!p || !p->X || !p->W) return fail(FQ3_ERR_INVALID, "null argument");
  if (p->T < 1 || p->Cin < 1 || p->N < 1 || p->taps < 1 || p->dil < 1 || p->batch < 0 || p->x_row0 < 0 || p->x_rows < 0)
    return fail(FQ3_ERR_INVALID, "T, Cin, N, taps and dil must be positive; batch, x_row0 and x_rows non-negative");
  if (p->mode < 0 || p->mode > 2) return fail(FQ3_ERR_INVALID, "mode must be 0 (general), 1 (SwiGLU) or 2 (GELU)");
  if (!p->Yraw && !p->Yact) return fail(FQ3_ERR_INVALID, "no output");
  if (p->mode == 1 && (p->Yact || p->R || p->bias || p->scale)) return fail(FQ3_ERR_INVALID, "the SwiGLU epilogue writes Yraw only");
  if ((p->bias && p->bias_mod < 1) || (p->scale && p->scale_mod < 1)) return fail(FQ3_ERR_INVALID, "bias_mod / scale_mod < 1");
  if (p->Yact && (!p->ea || !p->ib || p->act_mod < 1)) return fail(FQ3_ERR_INVALID, "Yact needs ea, ib and act_mod >= 1");
  fq3gemm::ConvArgs a;
  memset(&a, 0, sizeof(a));
  a.X = (const __nv_bfloat16*)p->X; a.W = (const __nv_bfloat16*)p->W; a.bias = p->bias; a.R = (const __nv_bfloat16*)p->R;
  a.Yraw = (__nv_bfloat16*)p->Yraw; a.Yact = (__nv_bfloat16*)p->Yact; a.ea = p->ea; a.ib = p->ib; a.scale = p->scale;
  a.T = p->T; a.Cin = p->Cin; a.N = p->N; a.taps = p->taps; a.dil = p->dil; a.mode = p->mode;
  a.bias_mod = p->bias ? p->bias_mod : 1; a.act_mod = p->Yact ? p->act_mod : 1; a.scale_mod = p->scale ? p->scale_mod : 1;
  a.x_row0 = p->x_row0; a.x_rows = p->x_rows; a.batch = p->batch;
  if (const char* err = fq3gemm::gemm(a, (cudaStream_t)stream)) return fail(FQ3_ERR_CUDA, "conv GEMM: %s", err);
  return 0;
}
