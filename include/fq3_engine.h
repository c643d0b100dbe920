/*
 * fq3_engine.h -- C ABI of the H100-native Qwen3-TTS decode engine.
 *
 * Drop-in boundary for the hot path of andimarafioti/faster-qwen3-tts.  The reference has no FFI on its torch
 * path (the seam is a Python duck type); the nearest precedent is the qwentts.cpp C ABI it reaches through
 * ctypes at faster_qwen3_tts/ggml_backend.py:216,381,446,499,645.  Each entry point below names the reference
 * interface it replaces (paths relative to the reference repo root).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no C++/torch types.
 *   - every function returns 0 on success, a negative fq3_status on failure; fq3_last_error() gives the text.
 *     Nothing throws across the ABI.
 *   - "dev" pointers are device memory owned by the caller (torch); the engine owns its packed weights, KV
 *     caches, scratch and per-request state.  `stream` is a cudaStream_t passed as void* (0 = default stream).
 *   - one engine per device; calls on one engine are not re-entrant; work is stream-ordered, the only host
 *     synchronisation is inside fq3_decode_chunk (it returns its result to host memory).
 *   - model dtype (FQ3_F32 / FQ3_BF16) is fixed at create time; all weight / activation tensors crossing the
 *     ABI are in that dtype, row-major, unless a parameter says otherwise.
 */
#ifndef FQ3_ENGINE_H
#define FQ3_ENGINE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct fq3_engine fq3_engine;

enum fq3_status {
  FQ3_OK = 0,
  FQ3_ERR_INVALID = -1,   /* bad argument / unsupported geometry           */
  FQ3_ERR_CUDA = -2,      /* CUDA runtime error                            */
  FQ3_ERR_STATE = -3,     /* call order violated (e.g. decode before load) */
  FQ3_ERR_TOO_LONG = -4   /* prompt longer than max_seq_len (talker_graph.py:163-167 raises RuntimeError) */
};

enum fq3_dtype { FQ3_F32 = 0, FQ3_BF16 = 1 };

/* One transformer stack (talker backbone or code predictor); fields mirror the HF config attributes the
 * reference reads (talker_graph.py:36-37,63-65; predictor_graph.py:41-46). head_dim is fixed at 128. */
typedef struct {
  int32_t hidden_size;
  int32_t intermediate_size;
  int32_t num_hidden_layers;
  int32_t num_attention_heads;
  int32_t num_key_value_heads;
  int32_t vocab_size;
  float rms_norm_eps;
} fq3_stack_config;

typedef struct {
  int32_t dtype;            /* fq3_dtype */
  int32_t device;           /* CUDA ordinal */
  int32_t max_seq_len;      /* talker KV capacity (model.py:113 default 2048); <= 4096 */
  int32_t num_code_groups;  /* 16 */
  int32_t codec_eos_token_id;
  int32_t has_mtp_projection; /* small_to_mtp_projection is a Linear (1.7B) or Identity (0.6B) */
  int32_t num_ctas;         /* 0 = one CTA per SM */
  int32_t rope_positions;   /* rows of the talker cos/sin tables (>= max_seq_len + margin for rope deltas) */
  fq3_stack_config talker;
  fq3_stack_config predictor;
  int32_t kv_pages;         /* talker KV page pool (see "Paged talker KV cache" below).  0 = max_slots *
                             * ceil(max_seq_len / 64) pages, slot s mapped for good to its own consecutive run; > 0 = a
                             * pool of that many pages, every slot unmapped; at least ceil(max_seq_len / 64) */
  int32_t max_batch;        /* columns one launch may carry (slots that advance together); 0/1 = one sequence, <= 32 */
  int32_t max_slots;        /* resident request slots (KV caches + per-request state); 0 = max_batch, else in
                             * [max_batch, FQ3_MAX_SLOTS].  Memory is the bound: fq3_slot_bytes() per slot */
} fq3_config;

/* Most request slots an engine may hold.  Beyond its memory a slot costs one host record, so the cap follows what an
 * 80 GB card holds: at the 1.7B geometry in bf16, 256 slots of max_seq_len 2048 are 60 GB of talker KV with the
 * default pool (a smaller kv_pages pool is what a slot then shares). */
#define FQ3_MAX_SLOTS 256

/* A named tensor handed to fq3_engine_load_weights.  Names (L = layers of that stack, stacked on dim 0):
 *   t.q [L,nH*128,H]  t.k [L,nKV*128,H]  t.v  t.o [L,H,nH*128]  t.gate [L,I,H]  t.up  t.down [L,H,I]
 *   t.ln_in [L,H]  t.ln_post [L,H]  t.qnorm [L,128]  t.knorm [L,128]  t.ln_f [H]
 *   t.head [V,H] (codec_head)   t.embed [V,H] (talker.get_input_embeddings())
 *   p.* likewise for the predictor, plus
 *   p.heads [15,Vp,Hp] (lm_head[i])   p.embeds [15,Vp,Ht] (codec_embedding[i])
 *   p.mtp_w [Hp,Ht]  p.mtp_b [Hp]     (only when has_mtp_projection)
 *   t.cos t.sin [rope_positions,128]  p.cos p.sin [32,128]   -- float32 always (HF rotary tables)
 * The engine copies / repacks; the caller may free the tensors afterwards. */
typedef struct {
  const char* name;
  const void* dev_ptr;
  int64_t numel;
} fq3_tensor;

/* Sampling parameters: sampling.py:32-66 (sample_logits) + sampling.py:10-29 (apply_repetition_penalty).
 * torch.multinomial is replaced by an inverse-CDF draw on caller-supplied uniforms (DESIGN.md, noise contract). */
typedef struct {
  int32_t do_sample;
  int32_t top_k;
  float temperature;
  float top_p;
  float repetition_penalty; /* talker only; 1.0 disables */
} fq3_sampling;

/* Request state set after prefill: generate.py:120-140 (first token, past_hidden, generation_step, prefill_len,
 * rope_deltas, left-pad count from attention_mask as in talker_graph.py:172-196). */
typedef struct {
  int32_t first_token;
  int32_t prefill_len;
  int32_t gen_step;
  int32_t rope_delta;
  int32_t n_left_pad;
  int32_t max_new_tokens;
  int32_t min_new_tokens;
  int32_t trailing_len;     /* rows of trailing_text_hiddens */
} fq3_request;

/* Why the on-device loop stopped (generate.py:149-151,175-177 and the for-range bound). */
enum fq3_finish { FQ3_RUNNING = 0, FQ3_FIN_MAX_NEW = 1, FQ3_FIN_EOS = 2, FQ3_FIN_MAX_SEQ = 3 };

/* A slot whose text is open (fq3_set_text_rows) stops at the frame that would read trailing row >= trailing_len, with
 * finished == FQ3_RUNNING: after a launch, finished == FQ3_RUNNING && frames_emitted < n_frames means "waiting for text".
 * The slot's state is then exactly what it is at an n_frames boundary, so the next launch resumes it unchanged. */
typedef struct {
  int32_t frames_emitted;   /* frames written by the last fq3_decode_chunk */
  int32_t finished;         /* fq3_finish */
  int32_t total_frames;     /* frames emitted since fq3_begin_request */
  int32_t next_token;       /* current cb0 token (the one the next frame would start from) */
} fq3_chunk_result;

/* ---- lifecycle ------------------------------------------------------------------------------------------ */
/* replaces TalkerGraph.__init__ / PredictorGraph.__init__ (talker_graph.py:27-59, predictor_graph.py:34-78):
 * allocates KV caches, scratch and tables.  A configuration that cannot succeed (max_slots < max_batch, max_slots >
 * FQ3_MAX_SLOTS, max_batch > 32, unsupported geometry) is refused with FQ3_ERR_INVALID before anything is allocated.
 * Every allocation is made before the first memset: when one does not fit, the call returns FQ3_ERR_CUDA, has freed
 * what it allocated, has launched nothing and leaves *out untouched. */
int fq3_engine_create(const fq3_config* cfg, fq3_engine** out);
/* Device bytes one resident request slot costs under `cfg` (talker and predictor K and V caches, loop state, past
 * hidden, penalty bitmap): the part of fq3_engine_create's allocation that grows with max_slots.  Pure arithmetic, no
 * device needed.  Negative fq3_status when cfg is NULL or its dtype is invalid. */
int64_t fq3_slot_bytes(const fq3_config* cfg);
/* Bytes of one talker KV page under `cfg` (2 * L * nKV * 64 * 128 * element size).  Pure arithmetic like
 * fq3_slot_bytes. */
int64_t fq3_kv_page_bytes(const fq3_config* cfg);
/* replaces holding references to the upstream nn.Modules (predictor_graph.py:53-57, talker_graph.py:41):
 * copies norm/embedding tables and repacks every GEMV weight into the per-CTA streaming tape. */
int fq3_engine_load_weights(fq3_engine* e, const fq3_tensor* tensors, int32_t n, void* stream);
void fq3_engine_destroy(fq3_engine* e);

/* Request slots.  The engine holds `max_slots` independent request slots (KV caches, predictor cache, penalty
 * bitmap, loop state).  Every per-request entry point names its slot, in [0, max_slots); fq3_decode_chunk takes the
 * list of at most `max_batch` slots that advance together: one slot runs the single-sequence persistent kernel,
 * several slots run the batched kernel in which all of them share ONE pass over the weight tape per step (the
 * reference batches left-padded prompts, model.py:774-787, with per-row pad counts, talker_graph.py:177-187).  A
 * column of a launch is a position in slots[], not a slot id: which resident slots a launch carries is the caller's
 * choice from launch to launch, and a slot that is not listed is not touched. */

/* Paged talker KV cache.  The talker's K/V rows live in pages of 64 rows taken from one engine-wide pool of
 * fq3_kv_pool_pages() pages.  A page is one contiguous block {K [L][nKV][64][128], V [L][nKV][64][128]} in model dtype.
 * Each slot has a page table: entry i is the page of its cache rows [64 i, 64 i + 64).  With the default pool
 * (kv_pages = 0) every slot is mapped to its own pages from creation on and nothing below is needed.
 * fq3_map_kv_pages sets slot's table to pages[0..n) (n <= ceil(max_seq_len / 64); n = 0 unmaps it).  Rows keep their
 * contents only where an entry keeps its page.  Refused before anything changes: a page outside the pool, a page listed
 * twice, a page mapped to another slot.  Returns once the table is on the device; no launch that reads the slot may
 * be in flight.  fq3_slot_kv_rows: the rows the slot's pages map (64 n).
 * No kernel touches an unmapped row: fq3_prefill[_batch] refuses P beyond the slot's rows, fq3_decode_chunk* a frame
 * budget whose frames would write past them, fq3_import_kv / fq3_export_kv P beyond them and fq3_talker_step a
 * position at or beyond them, all with FQ3_ERR_INVALID before launching anything. */
int fq3_map_kv_pages(fq3_engine* e, int32_t slot, const int32_t* pages, int32_t n);
int fq3_slot_kv_rows(fq3_engine* e, int32_t slot);
int fq3_kv_pool_pages(fq3_engine* e);
/* Whole pages pages[0..n) to / from caller memory (device or pinned host) [n][fq3_kv_page_bytes], stream-ordered,
 * one copy per page (parking a request's cache off the device).  Refused: a page outside the pool or listed twice. */
int fq3_kv_pages_to(fq3_engine* e, const int32_t* pages, int32_t n, void* dst, void* stream);
int fq3_kv_pages_from(fq3_engine* e, const int32_t* pages, int32_t n, const void* src, void* stream);

/* ---- duck-type compatibility path (what the reference's own schedulers call) ----------------------------- */
/* TalkerGraph.prefill_kv (talker_graph.py:153-170): k,v are [n_kv, P, 128] contiguous for one layer. */
int fq3_import_kv(fq3_engine* e, int32_t slot, int32_t layer, const void* k_dev, const void* v_dev, int32_t P,
                  void* stream);
/* inverse of fq3_import_kv: cache rows [0,P) of one layer -> k,v [n_kv, P, 128] (what a caller holding the
 * reference's StaticCache would read back; used by the parity tests of the hand-written prefill) */
int fq3_export_kv(fq3_engine* e, int32_t slot, int32_t layer, void* k_dev, void* v_dev, int32_t P, void* stream);
/* TalkerGraph.set_generation_state (talker_graph.py:172-196): per-row left-pad count and rope delta. */
int fq3_set_generation_state(fq3_engine* e, int32_t slot, int32_t n_left_pad, int32_t rope_delta);
/* TalkerGraph.run (talker_graph.py:198-214): one token through 28 layers + final norm.
 * embeds_dev [H] -> hidden_out_dev [H], both model dtype. */
int fq3_talker_step(fq3_engine* e, int32_t slot, const void* embeds_dev, int32_t position, void* hidden_out_dev,
                    void* stream);
/* PredictorGraph.run (predictor_graph.py:204-214): pred_input_dev [2,H_talker] -> codes_out_dev int64[15].
 * uniforms_dev float32[15] (ignored when !do_sample). */
int fq3_predictor_run(fq3_engine* e, int32_t slot, const void* pred_input_dev, const fq3_sampling* sp,
                      const float* uniforms_dev, int64_t* codes_out_dev, void* stream);
/* sampling.py:32-66 + :10-29 on a single logits row (model dtype, [V]); history_dev int64[n_hist] or NULL.
 * suppress range is [V-1024,V) except eos when suppress_special != 0 (generate.py:46-50). token_out_dev int64[1]. */
int fq3_sample_logits(fq3_engine* e, const void* logits_dev, int32_t V, const fq3_sampling* sp, float u,
                      const int64_t* history_dev, int32_t n_hist, int32_t suppress_special, int32_t eos_id,
                      int32_t suppress_eos, int64_t* token_out_dev, void* stream);
/* fq3_sample_logits (its NULL case) that also writes the log-probability of the drawn id to logprob_out_dev float32[1]
 * when it is not NULL, as fq3_decode_chunk_lp defines it; the first cb0 token of a request needs it.  The draw is
 * bit-identical with and without it. */
int fq3_sample_logits_lp(fq3_engine* e, const void* logits_dev, int32_t V, const fq3_sampling* sp, float u,
                         const int64_t* history_dev, int32_t n_hist, int32_t suppress_special, int32_t eos_id,
                         int32_t suppress_eos, int64_t* token_out_dev, float* logprob_out_dev, void* stream);

/* ---- K3: hand-written prefill (bf16 engines) ------------------------------------------------------------------ */
/* Borrow row-major weights for the prompt GEMMs (caller keeps them alive, 16-byte aligned): t.qkv [L,(nH+2nKV)*128,H]
 * (q,k,v rows concatenated), t.o [L,H,nH*128], t.gu [L,2I,H] (gate/up rows interleaved), t.down [L,H,I], t.head [V,H].
 * Requires H <= 2048, H % 32 == 0, I % 32 == 0, V % 8 == 0 and nH / nKV in {1, 2}. */
int fq3_engine_set_prefill_weights(fq3_engine* e, const fq3_tensor* tensors, int32_t n);
/* talker.forward prefill (generate.py:107-118) + TalkerGraph.prefill_kv (talker_graph.py:153-170) in one call:
 * embeds_dev [P,H] -> KV cache slots [0,P) of request slot `slot`, logits_out_dev [V] (16-byte aligned; codec_head on the last
 * position), hidden_out_dev [H] (post-norm hidden of the last position = past_hidden).  Positions are
 * cache index - n_left_pad (clamped at 0); keys below n_left_pad are masked. */
int fq3_prefill(fq3_engine* e, int32_t slot, const void* embeds_dev, int32_t P, int32_t n_left_pad,
                void* logits_out_dev, void* hidden_out_dev, void* stream);
/* Batched prefill: n prompts into n distinct request slots with one chain of launches (fq3_prefill is the n = 1 case).
 * slots[n], P[n], n_left_pad[n] are HOST arrays; embeds_dev [sum P_b][H] holds the prompts packed row-major in list
 * order (prompt b at row P_0 + ... + P_{b-1}); logits_out_dev [n][V] (16-byte aligned) and hidden_out_dev [n][H] get
 * row b for prompt b.  The norms and GEMMs run on the packed rows; RoPE, the KV append and the attention map every row
 * and 32-query block back to its prompt, whose query blocks and key tiles start at its own row 0 / cache row 0.
 * Bit-exactness: for every listed slot the KV cache rows [0, P_b), its logits row and its hidden row are bit-identical
 * to fq3_prefill of that prompt into that slot alone; slots not listed are not touched.
 * Scratch holds max_seq_len rows: when sum P_b exceeds it, the prompts run as consecutive groups in list order, each
 * as many prompts as fit (one prompt of up to max_seq_len rows always does).  A group costs the launches of one
 * fq3_prefill.
 * Refused before anything is launched (no slot changes): n outside [1, max_batch] (prompts per call, whatever
 * max_slots is), a slot listed twice, and per row
 * what fq3_prefill refuses (slot out of range, P <= 0, P > max_seq_len = FQ3_ERR_TOO_LONG with the reference's
 * message); the message names the row when n > 1. */
int fq3_prefill_batch(fq3_engine* e, int32_t n, const int32_t* slots, const void* embeds_dev, const int32_t* P,
                      const int32_t* n_left_pad, void* logits_out_dev, void* hidden_out_dev, void* stream);

/* ---- fused path (the persistent on-device loop) ---------------------------------------------------------- */
/* generate.py:120-147 / streaming.py:76-104: latch per-request state of `slot`.  past_hidden_dev [H] model dtype;
 * trailing_text_dev [trailing_len,H], tts_pad_dev [H] model dtype (borrowed until the request ends);
 * uniforms_dev float32 [(max_new_tokens+1)*16]: row s+1 = draws of frame s (col 0 talker, 1..15 predictor). */
int fq3_begin_request(fq3_engine* e, int32_t slot, const fq3_request* rq, const void* past_hidden_dev,
                      const void* trailing_text_dev, const void* tts_pad_dev, const float* uniforms_dev,
                      const fq3_sampling* sp_talker, const fq3_sampling* sp_predictor, void* stream);
/* Incremental text input (the step-by-step text layout: frame s adds trailing row s to the talker input, tts_pad once
 * the rows run out).  Announces that rows [0, trailing_len) of the buffer latched by fq3_begin_request are valid, and
 * whether more may follow (open != 0).  While open, a frame that would read row >= trailing_len is not run: the slot
 * stops there (see fq3_chunk_result) instead of feeding tts_pad, which would tell the model the text has ended, so a
 * text-fed request sees exactly the inputs of the same request with all rows latched at once.  open == 0 closes the
 * text: from then on the slot behaves like any other request, and its trailing_len is final (it may already have fed
 * tts_pad past it).  fq3_begin_request resets the slot to closed-as-latched.
 * Legal after fq3_begin_request and between launches.  The caller must have latched a buffer that holds every row it
 * will ever announce, and writes new rows stream-ordered before the next fq3_decode_chunk on the same stream.
 * Refused: inactive slot (FQ3_ERR_STATE), trailing_len smaller than before (FQ3_ERR_INVALID), open after a close
 * (FQ3_ERR_STATE), a different trailing_len after a close (FQ3_ERR_STATE), trailing_len > 0 without a latched buffer
 * (FQ3_ERR_INVALID). */
int fq3_set_text_rows(fq3_engine* e, int32_t slot, int32_t trailing_len, int32_t open);
/* generate.py:149-199 / streaming.py:106-173 for up to n_frames frames of every listed slot in ONE kernel launch.
 * slots[n_slots] distinct slot ids that have a latched request; codes_out_dev int64 [n_slots][n_frames][16];
 * res[n_slots] (host).  n_slots == 1: single-sequence kernel; n_slots >= 2: batched kernel, the slots advance in
 * lock-step and stop independently (EOS / max_new_tokens / max_seq_len).  Synchronises the stream. */
int fq3_decode_chunk(fq3_engine* e, const int32_t* slots, int32_t n_slots, int32_t n_frames, int64_t* codes_out_dev,
                     fq3_chunk_result* res, void* stream);
/* fq3_decode_chunk (its NULL case) that also returns the log-probability of every code it draws: logprob_out_dev float32
 * [n_slots][n_frames][16] or NULL.  Column k >= 1 of frame f is codebook k (predictor pass k); column 0 is the cb0 token
 * sampled at the end of frame f, i.e. frame f + 1's cb0 or the EOS that ends the request (a frame cut off by max_seq_len
 * samples none and leaves column 0 unwritten).  The first cb0 of a request comes from fq3_sample_logits_lp.
 * Computed in fp32 from exactly the values the draw used:
 *   sampling: l = the processed row (dtype-rounded logits, repetition penalty, suppressed ids at -inf, / temperature
 *             rounded, top-k / top-p filtered); lp = (l_tok - max l) - log(sum exp(l - max l)), the max and sum the
 *             softmax before the draw reduces;
 *   greedy:   the log-softmax of the penalised, suppressed logits at the chosen id (no temperature).
 * Codes are bit-identical with and without logprob_out_dev.  Rows at or past a slot's frames_emitted are not written;
 * neither is anything of a slot not listed. */
int fq3_decode_chunk_lp(fq3_engine* e, const int32_t* slots, int32_t n_slots, int32_t n_frames, int64_t* codes_out_dev,
                        float* logprob_out_dev, fq3_chunk_result* res, void* stream);
/* fq3_decode_chunk_lp with a frame budget per slot: n_frames[n_slots] (HOST array, every entry > 0) -- slot j emits at
 * most n_frames[j] frames in this launch.  codes_out_dev int64 [n_slots][F][16] and logprob_out_dev float32
 * [n_slots][F][16] or NULL, F = the largest budget.  A slot that has used its budget leaves the launch as a slot that
 * waits for text does: the others go on, its state is what it is at a launch boundary, and the next launch resumes it
 * unchanged, so its codes do not depend on the budgets it was given.  After the launch frames_emitted ==
 * min(n_frames[j], frames to the request's end); rows at or past it are not written.  fq3_decode_chunk_lp is the case
 * of equal budgets.  Refused before anything is launched: n_slots outside [1, max_batch], a slot outside
 * [0, max_slots), a slot listed twice or without a request, a budget <= 0. */
int fq3_decode_chunk_n(fq3_engine* e, const int32_t* slots, int32_t n_slots, const int32_t* n_frames,
                       int64_t* codes_out_dev, float* logprob_out_dev, fq3_chunk_result* res, void* stream);
/* last post-norm talker hidden (generate.py:198 past_hidden) of `slot` -> dst_dev [H] model dtype */
int fq3_get_past_hidden(fq3_engine* e, int32_t slot, void* dst_dev, void* stream);
int fq3_max_batch(fq3_engine* e);   /* columns per launch */
int fq3_max_slots(fq3_engine* e);   /* resident request slots (>= fq3_max_batch) */
/* numerics probe of the batched GEMV: y[col][row] = W_seg[row,:] . x[col,:] for one weight segment of stack 0 (talker) /
 * 1 (predictor): which 0 qkv, 1 o_proj, 2 gate/up (out = model dtype [ncols][I] = silu(gate)*up), 3 down, 4 head
 * (predictor: layer = codebook).  x_dev model dtype [ncols][K]; out_dev float32 [ncols][rows] (which != 2). */
int fq3_debug_gemv(fq3_engine* e, int32_t stack, int32_t layer, int32_t which, int32_t ncols, const void* x_dev,
                   void* out_dev, void* stream);

/* ---- debugging / introspection ---------------------------------------------------------------------------- */
/* When enabled, the next talker step / predictor pass 0 dumps per-layer intermediates (float32) into an engine
 * buffer; fq3_debug_read copies `count` floats starting at `offset` to host memory.  Layout in DESIGN.md. */
int fq3_debug_enable(fq3_engine* e, int32_t on);
int fq3_debug_read(fq3_engine* e, int64_t offset, int64_t count, float* host_dst);
/* bytes of packed weight tape streamed per talker step / per predictor frame (algorithmic bytes, for bench) */
int fq3_tape_bytes(fq3_engine* e, int64_t* talker_step_bytes, int64_t* predictor_frame_bytes);
int fq3_num_ctas(fq3_engine* e);
/* number of kernels launched by this engine since creation (bench.py "gpu_launches") */
int64_t fq3_launch_count(fq3_engine* e);
/* numerics probe of the dense-layer GEMM shared by K3 and K4 (fq3gemm::gemm, csrc/fq3_gemm.cuh: implicit-GEMM causal
 * conv1d, taps = 1 is a linear layer, and its fused epilogues); needs no engine.  One launch with exactly these
 * arguments; the fields mirror fq3gemm::ConvArgs.  Device pointers: X bf16 [batch][x_rows, or T when x_rows == 0][Cin];
 * W bf16 [N][taps][Cin]; bias fp32 [bias_mod] or NULL; scale fp32 [scale_mod] or NULL; R bf16 [batch][T][N] or NULL;
 * Yraw bf16 [batch][T][N] (mode 1: [batch][T][N/2]) or NULL; Yact bf16 [batch][T][N] (SnakeBeta of Yraw) or NULL;
 * ea / ib fp32 [act_mod] (exp(alpha), 1 / (exp(beta) + 1e-9)), read when Yact is set.  batch 0 or 1 = one sequence.
 * A shape or alignment the kernel refuses (Cin % 32, N % 8, SwiGLU N % 32, 16-byte operands) returns FQ3_ERR_CUDA with
 * the kernel's message and launches nothing; a missing output or parameter array, a non-positive size or (mode 1) an
 * operand the SwiGLU epilogue ignores returns FQ3_ERR_INVALID. */
typedef struct {
  const void* X;
  const void* W;
  const float* bias;
  const void* R;
  void* Yraw;
  void* Yact;
  const float* ea;
  const float* ib;
  const float* scale;
  int32_t T, Cin, N, taps, dil;
  int32_t mode;             /* 0 general, 1 SwiGLU on (gate, up) column pairs, 2 general with exact GELU */
  int32_t bias_mod, act_mod, scale_mod;   /* column n reads bias[n % bias_mod], ea / ib [n % act_mod], scale[n % scale_mod] */
  int32_t x_row0, x_rows;   /* output row m of a sequence reads input rows x_row0 + m - shift, zero outside [0, x_rows) */
  int32_t batch;
} fq3_conv_probe;
int fq3_debug_conv_gemm(const fq3_conv_probe* p, void* stream);

/* ---- K4: codec decoder (replaces the cuDNN path under speech_tokenizer.decode, model.py:924,1093,1122)
 * geom = {device, hidden_size, decoder_dim, n_blocks, rate_0..rate_{n-1}}; hidden_size and decoder_dim >> n_blocks must
 * be multiples of 32.  fq3_codec_load_weights: the waveform stack.  Tensor names / layouts: csrc/fq3_codec.cu. */
typedef struct fq3_codec fq3_codec;
int fq3_codec_create(const int32_t* geom, int32_t n_geom, fq3_codec** out);
int fq3_codec_load_weights(fq3_codec* c, const fq3_tensor* tensors, int32_t n, void* stream);
/* The decoder's front end -- everything of speech_tokenizer.decode before conv_in: 16-codebook embedding mean,
 * sliding-window pre-transformer (RMSNorm, RoPE, layer scale, SwiGLU), 2 x (ConvTranspose k=s + ConvNeXt) -- as
 * hand-written kernels + the same wgmma GEMM.  geom = {Q, codebook_size, hidden, intermediate, n_heads, n_layers,
 * sliding_window, n_up, ratio_0 ..}; fgeom = {rms_norm_eps, rope_theta}.  Tensor names / layouts: csrc/fq3_codec.cu. */
int fq3_codec_load_frontend(fq3_codec* c, const int32_t* geom, int32_t n_geom, const float* fgeom, int32_t n_fgeom,
                            const fq3_tensor* tensors, int32_t n, void* stream);
/* speech_tokenizer.decode({"audio_codes": [batch,T,16]}) (model.py:924,1093,1122; SURVEY 8(b) fq3_codec_decode):
 * codes_dev int64 [batch][T][Q] -> pcm float32 [batch][T * total_upsample] clamped to [-1,1].  `batch` windows of equal
 * length share every launch; each has its own causal left padding.  No library kernel is launched.  Requires
 * fq3_codec_load_weights + fq3_codec_load_frontend. */
int fq3_codec_decode_codes(fq3_codec* c, const int64_t* codes_dev, int32_t batch, int32_t T, float* pcm_out_dev,
                           void* stream);
/* Stateful streaming decode (SURVEY 8(f) item 2; replaces the reference's Phase-1 re-decode of everything so far and
 * its 25-frame Phase-2 context window, model.py:1085-1135): a stream keeps, for every causal layer, the tail of that
 * layer's input (conv history rows, the last window-1 attention keys / values), so a chunk of T frames costs T frames.
 * The PCM of a stream equals the one-shot decode of the same codes (the decoder is causal).
 * fq3_codec_stream_decode: the next T frames of n_streams distinct streams in one set of launches; codes_dev int64
 * [n_streams][T][Q]; pcm_out_dev float32 [n_streams][T * total_upsample] or NULL (state warm-up only, e.g. the ICL
 * reference frames). */
typedef struct fq3_codec_stream fq3_codec_stream;
int fq3_codec_stream_create(fq3_codec* c, fq3_codec_stream** out);
int fq3_codec_stream_reset(fq3_codec_stream* s, void* stream);
void fq3_codec_stream_destroy(fq3_codec_stream* s);
int64_t fq3_codec_stream_frames(fq3_codec_stream* s);
/* dst := src (layer histories + position), stream-ordered device copy: a stream warmed once with a voice reference is
 * the template of every later request that uses that reference */
int fq3_codec_stream_copy(fq3_codec_stream* dst, fq3_codec_stream* src, void* stream);
int fq3_codec_stream_decode(fq3_codec* c, fq3_codec_stream* const* streams, int32_t n_streams, const int64_t* codes_dev,
                            int32_t T, float* pcm_out_dev, void* stream);
double fq3_codec_flops(fq3_codec* c, int32_t T4);
double fq3_codec_frontend_flops(fq3_codec* c, int32_t T);
int64_t fq3_codec_launch_count(fq3_codec* c);
void fq3_codec_destroy(fq3_codec* c);
const char* fq3_codec_last_error(void);

/* ---- Speaking-rate control: pitch-preserving time-stretch of 24 kHz PCM on the device (csrc/fq3_tempo.cu)
 * WSOLA (waveform-similarity overlap-add) with a FQ3_TEMPO_WINDOW-sample periodic Hann window, synthesis hop
 * FQ3_TEMPO_WINDOW / 2 and a search of +-FQ3_TEMPO_SEARCH samples around each frame's nominal position; the score of a
 * candidate is its correlation with the previous frame's natural continuation over sqrt(FQ3_TEMPO_EPS + its energy).
 * The speed is quantised to q = round(speed * 1024) in [FQ3_TEMPO_Q_MIN, FQ3_TEMPO_Q_MAX]; q = 1024 is the identity and
 * has no tempo state (create refuses it: callers pass the PCM through).  The algorithm, bit for bit, is in DESIGN.md
 * ("Speaking rate") and faster_qwen3_tts/tempo.py.  A push releases exactly fq3_tempo_released(q, samples pushed before,
 * samples pushed now, flush) samples -- a function of the totals alone, so buffers are sized on the host and nothing is
 * read back.  The output of a stream depends on its samples and its flush point only, not on how they were pushed. */
#define FQ3_TEMPO_WINDOW 480
#define FQ3_TEMPO_SEARCH 240
#define FQ3_TEMPO_EPS 1e-6f
#define FQ3_TEMPO_Q_MIN 256
#define FQ3_TEMPO_Q_MAX 4096
typedef struct fq3_tempo fq3_tempo;
int fq3_tempo_create(int32_t device, double speed, fq3_tempo** out);
int fq3_tempo_reset(fq3_tempo* t);   /* a new stream at the same speed; host-side, nothing is launched */
void fq3_tempo_destroy(fq3_tempo* t);
/* samples released by a push of n samples after total_in (-1 for an invalid q or a negative count) */
int64_t fq3_tempo_released(int32_t q, int64_t total_in, int64_t n, int32_t flush);
/* One launch for n_streams distinct tempos.  in_dev float32: the streams' new samples packed in order (in_lens[i] of
 * stream i, host array); flush[i] (host) != 0 ends stream i (zeros after its end; it must be reset before more input).
 * out_dev float32 [out_cap]: the released samples packed in order; pk_dev int32 [pk_cap] or NULL: p_k of every frame run,
 * packed in order.  A null, misaligned or too small buffer, a tempo listed twice or a flushed tempo is refused before
 * anything is launched. */
int fq3_tempo_process(fq3_tempo* const* tempos, int32_t n_streams, const float* in_dev, const int64_t* in_lens,
                      const int32_t* flush, float* out_dev, int64_t out_cap, int32_t* pk_dev, int64_t pk_cap,
                      void* stream);
const char* fq3_tempo_last_error(void);

const char* fq3_last_error(void);
const char* fq3_version(void);

#ifdef __cplusplus
}
#endif
#endif /* FQ3_ENGINE_H */
