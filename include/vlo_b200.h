/*
 * vlo_b200.h — C ABI of libvlo_b200.so, the native CUDA engine (H100, sm_90a) for the per-frame hot
 * loop of showlab/videollm-online.
 *
 * The reference has no FFI: its seam is the Python duck-typed API of demo/inference.py and
 * models/*.py.  Each entry point below names the reference call it replaces (path:line relative
 * to the reference checkout, `HF:` = transformers 5.5).  INTEGRATION.md shows the ctypes binding
 * a maintainer of the reference would add.
 *
 * Conventions
 *  - every function returns 0 on success, a negative value on error; vlo_last_error() returns a
 *    thread-local message.  No exceptions cross the boundary.
 *  - pointers named d_* are raw DEVICE pointers (torch `tensor.data_ptr()`); h_* are host pointers.
 *    The engine never frees caller memory; the caller never frees engine memory.
 *  - `cuda_stream` is a cudaStream_t passed as void*; calls are asynchronous w.r.t. the host unless
 *    documented otherwise.
 *  - one engine per GPU/process; calls on one engine are not thread-safe (the Python host holds a lock).
 *  - 16-bit tensors: decoder/connector = bf16, vision tower = fp16 (the reference runs the ViT under
 *    fp16 autocast: models/modeling_live.py:23, models/vision_live.py:13).
 */
#ifndef VLO_B200_H_
#define VLO_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vlo_engine vlo_engine;

/* Model + capacity description.  Field meaning follows LlamaConfig / SiglipVisionConfig /
 * LiveConfigMixin (models/configuration_live.py:5-21). */
typedef struct vlo_config {
  /* decoder (Llama) */
  int32_t hidden_size, num_layers, num_heads, num_kv_heads, head_dim, intermediate_size, vocab_size;
  float rms_norm_eps;
  /* vision tower (SigLIP) */
  int32_t vit_hidden, vit_layers, vit_heads, vit_mlp, image_size, patch_size;
  float vit_ln_eps;
  /* frame tokens: frame_token_cls, frame_token_pooled (models/arguments_live.py:41-47) */
  int32_t frame_token_cls, pool_h, pool_w;
  /* capacities */
  int32_t max_streams;     /* concurrent video streams (KV caches) on this GPU */
  int32_t max_kv_tokens;   /* per-stream KV cap, tokens (the pool is shared: see vlo_engine_create_pooled) */
  int32_t max_step_tokens; /* max total new tokens in one vlo_step */
  int32_t max_vit_batch;   /* max frames per vlo_vit_encode */
} vlo_config;

/* Per-sequence result of a decoder step: everything demo/inference.py:76-81 and
 * models/modeling_live.py:177-179 read back from the logits, computed on the device. */
typedef struct vlo_decision {
  int32_t argmax_id;          /* plain greedy id (fast_greedy_generate) */
  int32_t argmax_excl_id;     /* argmax with the interval id removed (p(interval) < threshold case) */
  float p_interval;           /* softmax probability of the interval id, rounded to bf16 like the reference */
  float max_logit;            /* for diagnostics / margins */
  float top2_margin;          /* max logit - second max logit */
  float lse;                  /* log-sum-exp of the logits */
  int32_t argmax_prob_id;     /* argmax over the bf16-rounded softmax (what next_score.argmax sees), first index wins ties */
  int32_t reserved1;
} vlo_decision;

const char* vlo_last_error(void);
/* number of kernels of this library launched so far in this process (bench: gpu_launches) */
long long vlo_launch_count(void);
/* Optional CUDA-event profiler: when enabled every launch of the classes below is bracketed by an event
 * pair on its stream.  vlo_profile_read synchronises, returns per-class sums since the last read
 * (milliseconds, launches, algorithmic HBM bytes as defined in DESIGN.md) and resets.
 * classes: 0 weight-streaming GEMM (decoder/connector/lm_head), 1 KV-append attention, 2 split-KV merge,
 *          3 ViT GEMM, 4 ViT attention, 5 other. */
#define VLO_PROF_NUM_CLASSES 6
int vlo_profile_enable(int on);
int vlo_profile_read(double* ms, long long* launches, double* algo_bytes, int n_classes);
/* 1 when the device is an sm_90 (Hopper) part the kernels can run on */
int vlo_device_supported(int device);

/* ------------------------------------------------------------------ engine life cycle
 * replaces: build_live / LiveLlamaForCausalLM.from_pretrained + model.to('cuda')
 *           (models/modeling_live.py:184-222, demo/inference.py:15-16) */
int vlo_engine_create(const vlo_config* cfg, int device, vlo_engine** out);
/* KV cache = a pool of kv_pool_tokens (rounded up to whole 64-token pages) shared by all streams;
 * max_kv_tokens stays the per-stream cap.  kv_pool_tokens <= 0: max_streams * max_kv_tokens,
 * which is what vlo_engine_create reserves.  A stream holds ceil(kv_len / 64) pages; a step (or
 * vlo_kv_write / vlo_kv_copy_prefix / vlo_kv_fill_synthetic / vlo_kv_swap_in) that needs more pages than are
 * free fails with a "KV page pool exhausted" message.  Any of these calls that returns non-zero, for this or any
 * other reason, leaves every stream's kv_len and pages, and the free-page count, as they were before the call.
 * max_kv_tokens may not exceed 552 896 (the attention stages a split's page table in shared memory). */
int vlo_engine_create_pooled(const vlo_config* cfg, int64_t kv_pool_tokens, int device, vlo_engine** out);
int vlo_kv_pool_info(vlo_engine* e, int* page_tokens, int64_t* total_pages, int64_t* free_pages);
int vlo_engine_destroy(vlo_engine* e);
/* Register one weight tensor that already lives on the device in the ENGINE layout (see
 * DESIGN.md "weight layout"; the Python loader does the HF/peft key mapping, LoRA merge and
 * packing at init).  The engine keeps the pointer; the caller keeps the storage alive. */
int vlo_load_tensor(vlo_engine* e, const char* name, const void* d_ptr, int64_t n_bytes);
/* Resolve and size-check the registered tensors.  Each decoder layer matrix L{i}.{qkv,o,gate_up,down} comes in exactly
 * one form: bf16 `name`, or FP8 weights `name.f8` (e4m3fn bytes [N, K]) + `name.scale` (fp32 [N], one per row).  All
 * 4 x num_layers matrices must share one form; a mixed set, a missing scale or a wrong size fails with a message that
 * names the tensor.  The form decides which GEMM kernels the layer loop runs. */
int vlo_finalize_weights(vlo_engine* e);
/* bytes of device memory the engine allocated itself (KV + workspaces) */
int64_t vlo_engine_device_bytes(vlo_engine* e);

/* ------------------------------------------------------------------ streams (KV ownership)
 * replaces: the DynamicCache handed around as past_key_values (HF:cache_utils.py:88-121;
 *           demo/inference.py:47,69-70,91) */
int vlo_stream_open(vlo_engine* e, int* stream_id);
int vlo_stream_reset(vlo_engine* e, int stream_id);                 /* LiveInfer.reset: past_key_values = None */
int vlo_stream_close(vlo_engine* e, int stream_id);
int vlo_kv_len(vlo_engine* e, int stream_id, int* out_len);          /* Cache.get_seq_length() */
int vlo_kv_truncate(vlo_engine* e, int stream_id, int new_len);      /* trim_past_key_values(0, new_len), models/modeling_live.py:170-171 */
/* dst stream := the first n_tokens cache positions of src (device copy, all layers); dst's previous contents are dropped.
 * The engine-side form of `trim_past_key_values(past_key_values, 0, n)` when the ORIGINAL cache must survive
 * (stream_evaluate's look-ahead, models/modeling_live.py:112-113,170-171). */
int vlo_kv_copy_prefix(vlo_engine* e, int src_stream_id, int dst_stream_id, int n_tokens, void* cuda_stream);
/* Sliding window over a stream's cache (StreamingLLM): drop cache positions [first_token, first_token + n_tokens) and
 * move the later ones down by n_tokens, so positions stay contiguous.  first_token and n_tokens are multiples of the
 * page size (64), n_tokens > 0, and every dropped page is full: first_token + n_tokens <= 64 * floor(kv_len / 64).
 * The dropped pages leave the stream's table and go back to the pool; no row moves.  V rows are unchanged; every kept
 * K row after the dropped range is rotated in place by -n_tokens positions (one kernel over all layers and kv heads):
 *   k'[d]      = bf16(fl(fl(x1 * cos_d) + fl(x2 * sin_d)))
 *   k'[d + 64] = bf16(fl(fl(x2 * cos_d) - fl(x1 * sin_d)))        x1 = k[d], x2 = k[d + 64], d < head_dim / 2
 * with each fl one fp32 round-to-nearest (no FMA), cos_d / sin_d = h_cos[d] / h_sin[d] (host arrays of head_dim / 2
 * fp32 values: cos / sin of n_tokens * inv_freq[d], weights.rope_rotation).  Rows past kv_len on the last page are
 * left as they are.  The tables go through the pinned staging ring (no host synchronisation); the kernel is enqueued on
 * cuda_stream.  Ordering as vlo_kv_truncate: the stream is shorter on return, and the caller orders the call after the
 * work that wrote the stream and before work that reads it (usual stream / event rules).  A call that fails changes no
 * stream's length or table and no free-page count. */
int vlo_kv_evict(vlo_engine* e, int stream_id, int first_token, int n_tokens, const float* h_cos, const float* h_sin,
                 void* cuda_stream);
/* Token-granular window over a stream's cache: keep only the cache positions in n_spans spans
 * [keep_first[i], keep_first[i] + keep_len[i]) of stream_id (sorted, non-overlapping, each len > 0, inside [0, kv_len),
 * at least one position dropped).  Span i moves down to new_first[i] = sum_{j<i} keep_len[j]; its shift is
 * d_i = keep_first[i] - new_first[i].  V rows move unchanged.  K rows move and are rotated by -d_i with the exact formula
 * of vlo_kv_evict, using h_rot[i] = cos[head_dim/2] | sin[head_dim/2] of d_i (weights.rope_rotation), so h_rot holds
 * n_spans * head_dim fp32 values.  Rows with d_i = 0 are not touched.  The new kv_len is sum(keep_len).  Pages past
 * ceil(new_len / 64) go back to the pool; the rows past the new kv_len on the last page keep old, finite values.
 * The rows move in place, page by page in increasing order, through the decoder step's partial-sum workspace: the call
 * takes no free page and no device memory, and works on a full pool.  Because it uses that workspace it is ordered
 * like a step: enqueue it on the CUDA stream the engine's steps run on.  The tables go through one slot of the pinned
 * staging ring, which caps n_spans (hundreds at least; the error message of a larger call names the cap).  A call
 * that fails changes no stream's length, table or row and no free-page count. */
int vlo_kv_compact(vlo_engine* e, int stream_id, int n_spans, const int32_t* h_keep_first, const int32_t* h_keep_len,
                   const float* h_rot, void* cuda_stream);
/* test/bench hook: fill a stream's KV cache with deterministic pseudo-random values up to n_tokens
 * (pre-fill for the 12k-context measurements without replaying 1200 frames) */
int vlo_kv_fill_synthetic(vlo_engine* e, int stream_id, int n_tokens, uint64_t seed, void* cuda_stream);
/* copy one layer's K or V rows [n_kv_heads, len, head_dim] bf16 out of / into the cache (tests); d_out / d_in must be
 * 16-byte aligned (the copy moves 16 bytes per thread) */
int vlo_kv_read(vlo_engine* e, int stream_id, int layer, int is_v, void* d_out, void* cuda_stream);
int vlo_kv_write(vlo_engine* e, int stream_id, int layer, int is_v, const void* d_in, int n_tokens, void* cuda_stream);
/* Host images of a stream's cache, so an idle session can give its pages (and stream slot) back and resume later.
 * Image layout: [page j][layer][K|V][kv_head][64][128] bf16, pages in page-table order; page_bytes = n_kv_heads * 64 *
 * 128 * 2 (131 072 B for Llama-3-8B).  vlo_kv_image_bytes = ceil(n_tokens / 64) * 2 * num_layers * page_bytes.
 * The last page of an image also carries that page's rows past n_tokens: stale but finite pool rows, so the pool's
 * finiteness invariant (csrc/kv_pages.h) survives a round trip.
 * vlo_kv_swap_out: enqueues on cuda_stream one cudaMemcpy2DAsync per page (2 * num_layers rows of page_bytes at the
 * pool's plane stride; copy engines only, no kernel) into h_dst (pinned host memory of >= vlo_kv_image_bytes(kv_len)
 * bytes), then empties the stream: kv_len 0, pages released, slot still open.  The caller orders the copies after the
 * steps that wrote the stream (usual stream / event rules) and reads h_dst after them.
 * vlo_kv_swap_in: the stream must be open and empty; takes ceil(n_tokens / 64) pages (or fails with "KV page pool
 * exhausted" and changes nothing), enqueues the host-to-device copies from h_src (pinned) on cuda_stream and sets
 * kv_len = n_tokens.
 * Page reuse is ordered by the engine: pages released by a swap-out stay gated by an event recorded after its copies,
 * and any later call that takes such a page (a step, vlo_kv_write, vlo_kv_copy_prefix, vlo_kv_fill_synthetic,
 * vlo_kv_swap_in) makes its own cuda_stream wait on that event (cudaStreamWaitEvent; no host synchronisation).  Gated
 * pages count as free in vlo_kv_pool_info. */
int64_t vlo_kv_image_bytes(vlo_engine* e, int n_tokens);
int vlo_kv_swap_out(vlo_engine* e, int stream_id, void* h_dst, int64_t bytes, void* cuda_stream);
int vlo_kv_swap_in(vlo_engine* e, int stream_id, const void* h_src, int n_tokens, void* cuda_stream);

/* ------------------------------------------------------------------ hot path
 * vlo_vit_encode replaces LiveMixin.visual_embed (models/modeling_live.py:21-27) =
 *   _siglip_vision_encode (models/vision_live.py:10-30) + connector
 *   (models/live_llama/modeling_live_llama.py:18-22).
 * d_frames: uint8 [n_frames, 3, image, image]; d_out: bf16 [n_frames * frame_num_tokens, hidden].
 * d_vit_tokens (optional, may be NULL): fp32 [n_frames, frame_num_tokens, vit_hidden] = the
 * pre-connector tokens (what build_live_vision's encode_fn returns). */
int vlo_vit_encode(vlo_engine* e, const uint8_t* d_frames, int n_frames, void* d_out, float* d_vit_tokens,
                   void* cuda_stream);
/* connector only: visual_embed without a vision tower (models/modeling_live.py:22-27 with
 * pre-extracted features). d_tokens: bf16 [n_rows, vit_hidden] */
int vlo_connector(vlo_engine* e, const void* d_tokens, int n_rows, void* d_out, void* cuda_stream);
/* replaces model.get_input_embeddings()(ids) (demo/inference.py:46,66; models/modeling_live.py:181).
 * ids are clamped to vocab-1 like joint_embed does (models/modeling_live.py:38). */
int vlo_embed_tokens(vlo_engine* e, const int64_t* d_ids, int n, void* d_out, void* cuda_stream);
/* KV-append forward for a ragged batch — replaces LiveLlamaForCausalLM.forward(inputs_embeds=...,
 * past_key_values=..., use_cache=True) (models/live_llama/modeling_live_llama.py:24-67 ->
 * HF:models/llama/modeling_llama.py:375-499) plus the read of logits[:, -1:]
 * (demo/inference.py:76-81, models/modeling_live.py:177).
 *   h_stream_ids[n_seqs], h_q_lens[n_seqs]: host arrays; d_embeds: bf16 [sum(q_lens), hidden] packed.
 *   d_last_logits: bf16 [n_seqs, vocab] or NULL; d_decisions: vlo_decision[n_seqs] (device) or NULL.
 * Appends q_lens[i] tokens to stream i's KV cache. */
int vlo_step(vlo_engine* e, int n_seqs, const int32_t* h_stream_ids, const int32_t* h_q_lens, const void* d_embeds,
             void* d_last_logits, vlo_decision* d_decisions, int interval_id, void* cuda_stream);
/* Same, with token rows gathered on the device: d_row_ids[sum(q_lens)] (device int64), one entry per packed row;
 * id >= 0 = "this row is the embedding of token id" (gathered from the table, clamped to vocab-1),
 * id <  0 = "row already present in d_embeds" (a frame embedding).  The steady-state frame step is
 * [interval id, -1 x 10]; an AR step is [last id]; no separate embedding launch or torch.cat. */
int vlo_step_ids(vlo_engine* e, int n_seqs, const int32_t* h_stream_ids, const int32_t* h_q_lens,
                 const int64_t* d_row_ids, const void* d_embeds, void* d_last_logits, vlo_decision* d_decisions,
                 int interval_id, void* cuda_stream);
/* Segmented step: several decisions per sequence in one pass, e.g. a backlog of queued frames
 * [prefix | F1 | interval | F2 | interval | F3 ...] with one decision per frame.
 *   h_seg_counts[n_seqs] (host): sequence i carries h_seg_counts[i] >= 1 consecutive segments; their lengths follow one
 *   another in h_seg_lens (host, sum(h_seg_counts) entries, each > 0), and sequence i's q_len is the sum of its own.
 *   d_seg_logits: bf16 [sum(h_seg_counts), vocab] or NULL; d_decisions: vlo_decision[sum(h_seg_counts)] or NULL; one row
 *   per segment in order, computed at the segment's last row.
 * Each segment's attention is planned exactly as a one-sequence step of that segment alone over the keys up to its end
 * (same work items, split budget and key splits), so a segment computes the bits the same tokens get from a step of
 * their own on the same cache (decoder GEMM rows do not depend on the other rows of the step).  To take back the
 * segments after segment j, vlo_kv_truncate the stream to the end of segment j.  Row ids, page taking, pool-exhaustion
 * rollback and the capacity errors are those of vlo_step_ids, which is this call with one segment per sequence. */
int vlo_step_segments(vlo_engine* e, int n_seqs, const int32_t* h_stream_ids, const int32_t* h_seg_counts,
                      const int32_t* h_seg_lens, const int64_t* d_row_ids, const void* d_embeds, void* d_seg_logits,
                      vlo_decision* d_decisions, int interval_id, void* cuda_stream);
/* ------------------------------------------------------------------ response sampling
 * Replaces the logits processors HF's `generate(do_sample=True, ...)` runs per token (HF:generation/utils.py
 * GenerationMixin._get_logits_processor): RepetitionPenaltyLogitsProcessor, TemperatureLogitsWarper, TopKLogitsWarper,
 * TopPLogitsWarper, then a draw.  One vlo_sample_row per logits row; the kernel (csrc/sampling.cuh, sample_kernel)
 * applies, in fp32 on the bf16 logits and in this order:
 *   repetition penalty  l = l < 0 ? l * p : l / p for each distinct id of penalty_ids[offset, offset + count) (ids
 *                       outside [0, vocab) are ignored; p = 1: off);
 *   temperature         l = l / temperature;
 *   top-k               keep l >= the k-th largest l (ties kept; 0 or >= vocab: off);
 *   top-p               keep id i iff the softmax mass of the ids with a strictly larger probability is < top_p (>= 1:
 *                       off), over the top-k survivors.  A tie group straddling the boundary is kept whole (HF keeps
 *                       the part its sort puts first); the maximum is always kept;
 *   draw                id = first-index argmax over the kept i of l_i - log(-log(u_i)).
 * Noise layout (Philox4x32-10, 10 rounds, Random123 / curand constants): key = (seed & 0xffffffff, seed >> 32),
 *   counter = (i / 4, position, 0, 0) for vocab id i; word i % 4 of the output (x, y, z, w order) is x_i, and
 *   u_i = ((x_i >> 8) + 0.5) * 2^-24.  `position` is the stream position (KV row) of the token whose logits the row
 *   holds, so a row's id is a pure function of (logits, parameters): the same with any other rows in the launch, in
 *   a segmented verify step or in a one-token step, and in any run.
 * temperature 0: the row is not sampled (its id is -1). */
typedef struct vlo_sample_row {
  uint64_t seed;
  int32_t position;
  float temperature;         /* > 0; 0: skip the row */
  int32_t top_k;             /* 0: off */
  float top_p;               /* (0, 1); >= 1: off */
  float repetition_penalty;  /* > 0; 1: off */
  int32_t penalty_offset, penalty_count;  /* the row's ids in the call's penalty list (rows may share or overlap) */
  int32_t reserved;
} vlo_sample_row;
/* One id per row of d_logits (bf16 [n_rows, vocab], 16-byte aligned) into d_out_ids (device int32 [n_rows]), on
 * cuda_stream after the work before it (e.g. the vlo_step that wrote the logits).  n_rows <= max(max_streams,
 * max_step_tokens); n_penalty_ids <= 65 536.  The rows and the penalty ids (host arrays) go up through the engine's
 * pinned staging ring in one asynchronous copy: no host synchronisation. */
int vlo_sample(vlo_engine* e, const void* d_logits, int n_rows, const vlo_sample_row* h_rows, const int32_t* h_penalty_ids,
               int n_penalty_ids, int32_t* d_out_ids, void* cuda_stream);

/* all-position logits for the last vlo_step's tokens (the reference's logits_to_keep=0 behaviour,
 * HF:models/llama/modeling_llama.py:485-487); d_logits bf16 [sum(q_lens), vocab]. Test/compat path. */
int vlo_last_step_logits(vlo_engine* e, void* d_logits, void* cuda_stream);
/* final hidden states (post model.norm) of the last step, bf16 [sum(q_lens), hidden] (tests) */
int vlo_last_step_hidden(vlo_engine* e, void* d_hidden, void* cuda_stream);

/* ------------------------------------------------------------------ measurement hooks (bench.py roofline)
 * Back-to-back launches of one kernel class on the engine's own buffers: the KV-append attention over every
 * layer's cache of the given streams (n_tok query rows at the end of each cache; skip_merge = 1 leaves out the
 * split-KV merge kernel), and the four weight-streaming GEMMs
 * (qkv, o, gate_up, down) of every layer for n_tok token rows.  Asynchronous; the caller brackets the call with
 * CUDA events.  *h_algo_bytes = algorithmic HBM bytes per attention launch / per full pass over the layers. */
int vlo_bench_attn(vlo_engine* e, int n_seqs, const int32_t* h_stream_ids, int n_tok, int iters, int skip_merge,
                   double* h_algo_bytes_per_launch, void* cuda_stream);
int vlo_bench_gemm(vlo_engine* e, int n_tok, int iters, double* h_algo_bytes_per_iter, int* h_launches_per_iter,
                   void* cuda_stream);

/* ------------------------------------------------------------------ kernel-level entry points
 * (used by the parity tests and micro-benchmarks; same kernels the engine launches) */
/* One-tile GEMM of the ViT patch embed and MAP-head K/V projection (csrc/gemm.cuh), fp16:
 * y[t][n] = fp16(sum_k X[t,k] W[n,k] + bias[n]), X [rows_x, k], W [rows_w, k], k a multiple of 64;
 * epi 1: fp16 out[rows_x][ld_out] = act(y) (act codes in csrc/gemm.cuh);
 * epi 3: fp32 out[rows_x][ld_out] = y + pos[t % pos_rows][n], pos fp32 [pos_rows][ld_out].
 * bn = feature-tile width, 64 or 128 (0: 128). */
int vlo_op_gemm(int epi, int act, const void* d_x, int rows_x, const void* d_w, int rows_w, int k, void* d_out, int ld_out,
                const float* d_bias, const float* d_pos, int pos_rows, int bn, void* cuda_stream);
/* Persistent weight-streaming GEMM (csrc/gemm_ws.cuh): out[t, n] = sum_k X[t,k] W[n,k].  bn = token-tile width
 * (0: the smallest of 16/32/64/128 covering rows_x, with 96 too for bf16, and 128 above 128 rows; 64/96/128/192
 * tile larger rows_x).
 * mode 0: stream-K over all SMs, fp32 partial planes out[plane][rows_x][rows_w] (the caller zero-fills d_out
 *         and sums the planes; *h_max_planes tells how many planes to provide); d_out == NULL only plans.
 * mode 1: whole tiles, 16-bit out[rows_x][ld_out] = act(acc + bias). */
int vlo_op_gemm_ws(int fmt, int mode, const void* d_w, int rows_w, const void* d_x, int rows_x, int k, void* d_out,
                   int ld_out, long long plane_stride, const float* d_bias, int act, int n_ctas, int bn, int* h_max_planes,
                   void* cuda_stream);
/* The same GEMM in mode 0 on e4m3 weights (the decoder's FP8 weight form): d_w8 [rows_w, k] e4m3fn bytes, d_scale fp32
 * [rows_w] row scales, X bf16 [rows_x, k].  Same token tile and stream-K plan as the bf16 call with these sizes and
 * n_ctas; each weight k-block is upcast to bf16 exactly and multiplied by the bf16 wgmma chain, so plane p holds
 * fl(P_p[t][n] * d_scale[n]), P_p being plane p of the bf16 call on the upcast weights.  d_out == NULL only plans
 * (*h_max_planes).  Asynchronous. */
int vlo_op_gemm_ws_f8(const void* d_w8, const float* d_scale, int rows_w, const void* d_x, int rows_x, int k, float* d_out,
                      long long plane_stride, int n_ctas, int* h_max_planes, void* cuda_stream);
/* ViT trunk GEMM (csrc/gemm_vit.cuh), fp16, 128-token x 128-feature tiles:
 * out[t][n] = act(fp16(sum_k X[t,k] W[n,k] + bias[n])), fp16 out[rows_x][ld_out], ld_out even and >= rows_w;
 * n_ctas <= 0: one CTA per SM. */
int vlo_op_gemm_vit(const void* d_w, int rows_w, const void* d_x, int rows_x, int k, void* d_out, int ld_out,
                    const float* d_bias, int act, int n_ctas, void* cuda_stream);
/* KV-append attention over one layer's cache (the graded kernel, K15):
 *   d_q bf16 [n_tok, n_heads, head_dim] (RoPE applied); d_k/d_v bf16 [n_kv_heads, kv_stride, head_dim];
 *   keys 0..kv_len-1 valid, the n_tok query tokens sit at positions kv_len-n_tok .. kv_len-1 (causal with
 *   offset, HF:masking_utils.py:263-272); d_out bf16 [n_tok, n_heads*head_dim]; d_ws fp32 scratch of
 *   vlo_op_attn_ws_bytes(). Replaces HF:models/llama/modeling_llama.py:272-285 (SDPA / flash-attn 2). */
int64_t vlo_op_attn_ws_bytes(int n_tok, int n_heads, int head_dim, int kv_len);
int vlo_op_attn_kvappend(const void* d_q, const void* d_k, const void* d_v, void* d_out, float* d_ws, int n_tok,
                         int n_heads, int n_kv_heads, int head_dim, int kv_len, long long kv_stride, void* cuda_stream);
/* kernel-level: the decoder attention over a paged pool [n_pages, n_kv_heads, 64, 128] (tests).  d_page_table: device
 * int32 [ceil(kv_len / 64)], the page of each 64-key block; other arguments as vlo_op_attn_kvappend.  Rows of the last
 * page past kv_len must be finite. */
int vlo_op_attn_kvappend_paged(const void* d_q, const void* d_k_pool, const void* d_v_pool, const int32_t* d_page_table,
                               int n_pages, void* d_out, float* d_ws, int n_tok, int n_heads, int n_kv_heads,
                               int head_dim, int kv_len, void* cuda_stream);
/* kernel-level: the attention of one segmented sequence over a paged pool, planned and launched as vlo_step_segments
 * does.  n_tok = sum(h_seg_lens[0..n_segs)) query rows (host array, each > 0) sit at positions kv_len - n_tok ..
 * kv_len - 1 of d_q [n_tok, n_heads, head_dim]; row r attends causally to keys 0..(its position).  Segment j (rows
 * o_j .. o_j + len_j - 1, ending at key e_j = kv_len - n_tok + o_j + len_j) gets in d_out exactly the bits
 * vlo_op_attn_kvappend_paged gives its rows alone with kv_len = e_j on the same pool.  n_segs = 1 is that call.
 * Keys past a row's position are masked: they may hold any finite values.  Scratch is allocated internally;
 * synchronous. */
int vlo_op_attn_kvappend_segments(const void* d_q, const void* d_k_pool, const void* d_v_pool, const int32_t* d_page_table,
                                  int n_pages, void* d_out, int n_segs, const int32_t* h_seg_lens, int n_heads,
                                  int n_kv_heads, int head_dim, int kv_len, void* cuda_stream);
/* The attention plan vlo_op_attn_kvappend_segments (and vlo_step_segments, for one sequence) makes for these segments,
 * without launching anything: h_counts[0..4) = work items, 2-CTA clusters, packs (runs of consecutive one-token
 * segments one CTA per (split, kv head) computes in one pass over the cache) and the items inside packs.  Queries the
 * current device's SM count. */
int vlo_op_attn_plan_counts(int n_segs, const int32_t* h_seg_lens, int n_heads, int n_kv_heads, int head_dim, int kv_len,
                            int32_t* h_counts);
/* The ViT attention kernels of vlo_vit_encode (csrc/vit_kernels.cuh), launched by the same helpers; fp16 tensors,
 * head_dim 64, hidden = 64 x heads, n_frames frames of n_tok tokens.  Asynchronous.
 * vit_attn: d_qkv [n_frames * n_tok, 3 * hidden] (q | k | v column blocks, head h at columns 64 h .. of each) ->
 *   d_out [n_frames * n_tok, hidden] = softmax(q k^T / 8) v over the keys of the query's own frame, per head.
 * probe_attn (the MAP head): d_kv [n_frames * n_tok, 2 * hidden] (k | v), d_q fp32 [hidden] one query shared by every
 *   frame -> d_out [n_frames, hidden] = softmax(q k^T / 8) v per head and frame; n_tok <= 12288. */
int vlo_op_vit_attn(const void* d_qkv, void* d_out, int n_frames, int n_tok, int hidden, void* cuda_stream);
int vlo_op_probe_attn(const void* d_kv, const float* d_q, void* d_out, int n_frames, int n_tok, int hidden,
                      void* cuda_stream);
/* The decoder step's fix-up and decision kernels (csrc/decoder_kernels.cuh), launched by the same helpers as vlo_step
 * (block size, grid, shared memory, PDL).  bf16 tensors unless stated; bf16(.) = round to nearest even.
 * d_part: fp32 stream-K partial planes [plane][T][width] as vlo_op_gemm_ws mode 0 leaves them (plane_stride T * width)
 * for the bf16 GEMM of `width` output features over T token rows with this k and n_ctas (<= 0: one CTA per SM).  The
 * entries take the plan from that GEMM's planning query and read only the sk_planes(tile) planes of each 128-feature
 * tile (csrc/streamk.h).  They reject T > 128 (one token tile) and plans of more than 8 planes.
 * Fix-up of feature n of token t: y = bf16(sum_{s < planes(n / 128)} part[s][t][n]), summed in plane order in fp32. */
/* Residual add + RMSNorm, width = H (a multiple of 4, <= 12288):
 *   h[t] = bf16(h[t] + y[t])                        (d_part == NULL: no partials, h unchanged)
 *   xn[t][i] = bf16(w[i] * bf16(h[t][i] * rsqrt(mean_i(h[t][i]^2) + eps)))   (d_xn may be NULL)
 *   xn_last[last_index[t]] = xn[t] for every t with last_index[t] >= 0      (d_last_index / d_xn_last may be NULL)
 * Asynchronous. */
int vlo_op_resid_rmsnorm(const float* d_part, int k, int n_ctas, void* d_h, const void* d_w, void* d_xn, void* d_xn_last,
                         const int32_t* d_last_index, int T, int H, float eps, void* cuda_stream);
/* q|k|v fix-up + RoPE + KV append, width = (n_heads + 2 n_kv_heads) * 128, head hh = features [128 hh, 128 hh + 128):
 * heads < n_heads are q, then n_kv_heads k heads, then n_kv_heads v heads.  For d < 64, x1 = y[d], x2 = y[d + 64]:
 *   q and k: out[d] = bf16(bf16(x1 c) + bf16(-x2 s)), out[d + 64] = bf16(bf16(x2 c) + bf16(x1 s)),
 *            c = cos[pos][d], s = sin[pos][d] (bf16 tables [n_rope_pos][64]); v: out = y unrotated.
 *   q heads -> d_q [T, n_heads, 128]; kv head j -> row h_tok_kvrow[t] + j * kv_head_stride of d_k / d_v (rows of 128).
 * h_tok_pos / h_tok_kvrow: host arrays [T]; every position must lie in [0, n_rope_pos).  Synchronous. */
int vlo_op_qkv_rope_append(const float* d_part, int k, int n_ctas, const void* d_cos, const void* d_sin, int n_rope_pos,
                           const int32_t* h_tok_pos, const int64_t* h_tok_kvrow, int kv_head_stride, void* d_q, void* d_k,
                           void* d_v, int T, int n_heads, int n_kv_heads, void* cuda_stream);
/* Fused gate|up GEMM + SwiGLU (csrc/gemm_wsf.cuh), the decoder's: W [rows_w, k] with rows_w % 128 == 0, 128-row tile j
 * = 64 gate rows then the matching 64 up rows (features 64 j ..); X [rows_x <= 128, k].  With g, u = bf16 of the fp32
 * stream-K sums over all SMs,  act[t][64 j + i] = bf16(bf16(g / (1 + exp(-g))) * u),  act [rows_x, rows_w / 2].
 * d_planes: fp32 scratch of plane_elems floats for the partials; d_flags: n_flags >= rows_w / 128 int32 arrival
 * counters, zero before the call and zero again when it has run.  Asynchronous. */
int vlo_op_gemm_swiglu(const void* d_w, int rows_w, const void* d_x, int rows_x, int k, void* d_act, float* d_planes,
                       int64_t plane_elems, int32_t* d_flags, int n_flags, void* cuda_stream);
/* vlo_op_gemm_swiglu on e4m3 weights d_w8 [rows_w, k] with fp32 row scales d_scale [rows_w] (same row order and plan):
 * g, u = bf16(sum_p fl(P_p * d_scale[n])) summed in plane order, P_p the fp32 partials of the bf16 kernel on the exactly
 * upcast weights (the finisher's own partial is plane 0).  Asynchronous. */
int vlo_op_gemm_swiglu_f8(const void* d_w8, const float* d_scale, int rows_w, const void* d_x, int rows_x, int k, void* d_act,
                          float* d_planes, int64_t plane_elems, int32_t* d_flags, int n_flags, void* cuda_stream);
/* Speak / silent decision over bf16 logits [n_rows, vocab] (vocab a multiple of 8, rows 16-byte aligned), one
 * vlo_decision per row into d_out (device): first-index argmax, max logit, max - second max (a repeated maximum counts
 * as the second), log-sum-exp, p_interval = bf16(softmax[interval_id]) (0 when interval_id is outside the row), and the
 * first-index argmax of bf16(softmax) with (argmax_prob_id) and without (argmax_excl_id: that entry set to 0) the
 * interval id.  Asynchronous. */
int vlo_op_decision(const void* d_logits, int n_rows, int vocab, int interval_id, vlo_decision* d_out, void* cuda_stream);
/* The sampling kernel of vlo_sample without an engine (any vocab % 8 == 0).  d_info (device, may be NULL): per row
 * {int32 kept count, float top-k threshold, float top-p threshold, int32 0}: an id is kept iff its l (after penalty and
 * temperature) is >= both thresholds (-inf: that filter is off).  Parameters are uploaded from pageable memory;
 * synchronous. */
int vlo_op_sample(const void* d_logits, int n_rows, int vocab, const vlo_sample_row* h_rows, const int32_t* h_penalty_ids,
                  int n_penalty_ids, int32_t* d_out_ids, void* d_info, void* cuda_stream);
/* Micro-loop of the same attention over n_layers separate K / V matrices (working set > L2), iters passes of back-to-back
 * launches on one plan: what bench tools bracket with ONE CUDA-event pair (per-launch time incl. the PDL overlap of a real
 * step).  skip_merge != 0 launches the main kernel only.  Mirrors vlo_bench_attn without an engine. */
int vlo_op_attn_bench(const void* d_q, const void* d_k, const void* d_v, void* d_out, float* d_ws, int n_tok, int n_heads,
                      int n_kv_heads, int head_dim, int kv_len, long long kv_stride, int n_layers,
                      long long layer_stride_rows, int iters, int skip_merge, double* h_algo_bytes, void* cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* VLO_B200_H_ */
