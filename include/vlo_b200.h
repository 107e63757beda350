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
 * one form: bf16 `name`, or FP8 weights `name.f8` (e4m3fn bytes [N, K]) + `name.scale` (fp32 [N], one per row), or int4
 * weights `name.i4` + `name.gscale`.  All 4 x num_layers matrices must share one form; a mixed set, a missing scale or a
 * wrong size fails with a message that names the tensor.  The form decides which GEMM kernels the layer loop runs.
 * The int4 form (W4A16, weights.quantize_int4_groups), groups of 128 along K (K % 128 == 0, else finalize fails):
 *   s[n, g] = bf16_rn(fp32(max_{k in g} |W[n,k]|) / 7), 1 where that is 0;  q[n, k] = clamp(rne(fp32(W) / fp32(s)), -8, 7);
 *   the weight every kernel multiplies is W4[n, k] = bf16_rn(q * s) (q * s is exact in fp32: one rounding).
 * `name.gscale` is bf16 [N, K / 128].  `name.i4` holds the codes q + 8, two per byte, ceil(N / 128) x 128 x K / 2 bytes in
 * the engine byte order: one 4 KB block per (128-row tile, 64-wide k-block), blocks in (tile, k-block) order, and inside a
 * block thread t of the consumer warpgroup's 16 bytes per 64-row half h at h * 2048 + 16 t (DESIGN.md section 2,
 * weights.pack_int4_codes).  Every result is bit for bit the bf16 engine's on W4.  An int4 engine prefills only with
 * vlo_set_quantized_prefill (vlo_max_prefill_tokens is 0 without it) and takes no FP8 activations (finalize fails with a
 * message).
 * The vocabulary matrices `embed` and `lm_head` ([vocab, hidden] each) come either in bf16 (`embed`, `lm_head`) or, on
 * an engine with quantized layer matrices, both in the layers' quantized form, quantized by the same rules:
 *   int4 layers: `embed.i4` + `embed.gscale`, `lm_head.i4` + `lm_head.gscale` (engine byte order, as above).  lm_head
 *     writes bf16(acc), acc the bf16 lm_head's fp32 chain over W4; the embedding of id i is row i of W4.  Every result is
 *     bit for bit that of the same int4 engine loaded with the dequantized vocabulary matrices in bf16.
 *   e4m3 layers (also with FP8 activations): `embed.f8` + `embed.scale`, `lm_head.f8` + `lm_head.scale`.  lm_head
 *     multiplies the bf16 final-norm rows by the exactly upcast codes (bf16 MMAs) and writes bf16(fl(acc * s[n])); the
 *     embedding of id i is bf16_rn(fp32(q[i, k]) * s[i]).
 * Finalize fails with a message on a vocabulary matrix in the other quantized form, on embed and lm_head in different
 * forms, on quantized vocabulary matrices next to bf16 layers, and on missing or wrongly sized tensors.  A failed
 * finalize leaves the previous tables untouched.  vlo_vocab_format tells the form the engine loaded. */
int vlo_finalize_weights(vlo_engine* e);
/* GemmFmt of the vocabulary matrices the last successful vlo_finalize_weights installed: 1 bf16, 2 e4m3, 4 int4; -1
 * before one with a decoder.  A failed finalize does not change it. */
int vlo_vocab_format(vlo_engine* e);
/* bytes of device memory the engine allocated itself (KV + workspaces) */
int64_t vlo_engine_device_bytes(vlo_engine* e);
/* FP8 activations (W8A8), on top of FP8 layer weights.  Valid before vlo_finalize_weights (fails after it); finalize then
 * fails with a message if the mode is on and the layer matrices are bf16.  on != 0 allocates the e4m3 activation copies
 * (max_step_tokens x (hidden + heads x head_dim + intermediate) bytes plus three fp32 scales per token); a default
 * engine never holds them.  Numerics of the mode, for each of the four layer GEMMs:
 *   - the activation operand is the bf16 tensor the FP8-weight path multiplies: xn after the input RMSNorm (q|k|v), the
 *     attention output (o_proj), xn after the post-attention RMSNorm (gate|up), the SwiGLU output act (down_proj);
 *   - per token row t it is quantized as weights.quantize_fp8_rows quantizes a weight row:
 *       a_s[t] = fp32(max_k |X[t,k]|) / 448 (1 for an all-zero row),
 *       q[t,k] = e4m3fn(clamp(fp32(X[t,k]) / a_s[t], +-448)), IEEE fp32 division, rounded to nearest even;
 *   - contributor p of a tile writes fl(fl(P_p[t][n] * w_s[n]) * a_s[t]) into its plane, P_p the e4m3 x e4m3 products
 *     summed over that CTA's k-blocks by the FP8 wgmma chain, whose accumulation is not full IEEE fp32 (exact only while
 *     the partial sums are small integers); the fix-up kernels and the gate|up finisher add the planes as before.
 * The lm_head, embedding, norms, residual stream, RoPE, KV cache, connector and ViT keep their formats; xn (hence
 * xn_last and vlo_last_step_hidden) is still written in bf16.  Two more launches per layer: the quantizers of the
 * attention output and of act (the norms write the e4m3 xn themselves). */
int vlo_set_fp8_activations(vlo_engine* e, int on);
/* Prefill on quantized layer matrices (FP8 weights, W8A8, int4), opt-in.  Valid before vlo_finalize_weights (fails after
 * it).  With on != 0, finalize grows the token-row workspaces to vlo_max_prefill_tokens rows as it does on a bf16 engine
 * and, under FP8 activations, the e4m3 activation copies and their token scales too; vlo_prefill then runs the layer
 * GEMMs on gemm_prefill_q_kernel (csrc/gemm_prefill_q.cuh), with the bits of the same rows fed as max_step_tokens steps
 * on the same engine.  Finalize fails with a message if the mode is on and the layer matrices are bf16 (a bf16 engine
 * always prefills).  Off (the default), a quantized engine keeps its workspaces at max_step_tokens rows and does not
 * prefill. */
int vlo_set_quantized_prefill(vlo_engine* e, int on);

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
 * ceil(new_len / 64) go back to the pool; the rows past the new kv_len on the last page keep their old values.
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
 * The last page of an image also carries that page's rows past n_tokens: stale pool rows.  They are masked rows of the
 * attention and may hold anything, non-finite values included.
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
/* vlo_letterbox replaces the host preprocessing of a clip: ffmpeg_once's `scale` + `pad` to image x image (data/utils.py:51-66,
 * called from demo/cli.py:15-20), which video_ingest.read_video_resampled applies with OpenCV's INTER_CUBIC.  It turns
 * n_frames native frames, each of its own size, into the canvases vlo_vit_encode reads: d_out uint8
 * [n_frames, 3, image, image], RGB.  One descriptor per frame (host array, passed to the kernel by value):
 *   d_pixels   uint8 [height][width][3], packed, RGB or BGR (bgr != 0);
 *   1 <= width, height <= 8192;
 *   d_taps     int32 tap tables (16-byte aligned): the horizontal table starts at row x_taps, the vertical one at row
 *              y_taps; a row is {i0, i1, i2, i3, w0, w1, w2, w3}, one per output column (sw rows) / line (sh rows).
 * Geometry: (sw, sh, x0, y0) = video_ingest.letterbox_geometry(width, height, image); every byte outside the scaled image
 * is 0 and every byte of the canvas is written.  The scaled pixel (dx, dy), channel c, is
 *   h_k = sum_j src[iy_k][ix_j][c] * wx_j   (int32; i = the row's indices clamped to the image, w = its weights)
 *   v   = sum_k h_k * wy_k                  (int32)
 *   out = clamp((v + 2^21) >> 22, 0, 255)
 * which is OpenCV's fixed-point INTER_CUBIC when the tables are video_ingest.cubic_taps (11-bit weights of A = -0.75).
 * Checks null pointers, sizes, n_frames <= max_vit_batch, the table alignment and that bgr is 0 or 1; one launch per 48
 * frames, asynchronous, ordered behind the previous work on cuda_stream (the canvas may still be read by it). */
typedef struct vlo_letterbox_frame {
  const uint8_t* d_pixels;
  const int32_t* d_taps;
  int32_t width, height, bgr;
  int32_t x_taps, y_taps;
  int32_t reserved;
} vlo_letterbox_frame;
int vlo_letterbox(vlo_engine* e, const vlo_letterbox_frame* h_frames, int n_frames, uint8_t* d_out, void* cuda_stream);
/* vlo_letterbox_planes is vlo_letterbox for frames given as planes, as camera and decoder pipelines deliver them: the
 * same geometry, tap tables, integer INTER_CUBIC and canvases, with each source pixel converted to RGB where the cubic
 * sums read it.  One descriptor per frame; a launch may mix formats and sizes.  format (plane p at d_planes[p], row r of
 * it at d_planes[p] + r * pitch[p], pitch[p] >= the plane's row bytes; padding past the row bytes is never read):
 *   VLO_PIX_RGB24 / VLO_PIX_BGR24  1 plane  uint8 [height][width][3] packed           (1 <= width, height <= 8192)
 *   VLO_PIX_NV12                   2 planes Y [height][width], UV [height/2][width/2][2] interleaved
 *   VLO_PIX_I420                   3 planes Y [height][width], U [height/2][width/2], V [height/2][width/2]
 *   VLO_PIX_YUYV                   1 plane  [height][width/2] pairs {Y0, U, Y1, V}     (ffmpeg's yuyv422)
 * The YUV formats take 2 <= width, height <= 8192, width even, height even for NV12 and I420.  Pixel (x, y) has luma
 * Y = its Y sample and chroma U, V = the sample of (x/2, y/2) (NV12, I420) or of pair x/2 (YUYV), taken nearest; it
 * enters the cubic sums as OpenCV's fixed-point BT.601 limited-range cvtColor(COLOR_YUV2RGB_NV12 / _I420 / _YUYV):
 *   y = max(Y - 16, 0) * 1220542,  u = U - 128,  v = V - 128
 *   R = clamp((y + 2^19 + 1673527 v) >> 20, 0, 255)
 *   G = clamp((y + 2^19 - 852492 v - 409993 u) >> 20, 0, 255)
 *   B = clamp((y + 2^19 + 2116026 u) >> 20, 0, 255)
 * (int32, arithmetic shift).  The clamp precedes the cubic sums, so the canvas is exactly vlo_letterbox's canvas of
 * cvtColor's RGB frame.  Checks, before any launch, and leaves d_out untouched on failure: null planes, tables or output,
 * an unknown format, sides outside the limits above, odd sides, a pitch below the row bytes, the table alignment,
 * negative table offsets and n_frames in [1, max_vit_batch].  The descriptors travel as kernel parameters within the
 * 4 KB parameter space: one launch per 48 frames, asynchronous, ordered as vlo_letterbox. */
enum { VLO_PIX_RGB24 = 0, VLO_PIX_BGR24 = 1, VLO_PIX_NV12 = 2, VLO_PIX_I420 = 3, VLO_PIX_YUYV = 4 };
typedef struct vlo_frame_planes {
  const uint8_t* d_planes[3];   /* unused planes may be NULL */
  const int32_t* d_taps;        /* as vlo_letterbox_frame, tables of the luma width x height */
  int32_t pitch[3];             /* bytes from one row of a plane to the next */
  int32_t format, width, height;
  int32_t x_taps, y_taps;
} vlo_frame_planes;
int vlo_letterbox_planes(vlo_engine* e, const vlo_frame_planes* h_frames, int n_frames, uint8_t* d_out,
                         void* cuda_stream);
/* connector only: visual_embed without a vision tower (models/modeling_live.py:22-27 with
 * pre-extracted features). d_tokens: bf16 [n_rows, vit_hidden] */
int vlo_connector(vlo_engine* e, const void* d_tokens, int n_rows, void* d_out, void* cuda_stream);
/* replaces model.get_input_embeddings()(ids) (demo/inference.py:46,66; models/modeling_live.py:181).
 * ids are clamped to vocab-1 like joint_embed does (models/modeling_live.py:38).  With quantized vocabulary matrices the
 * rows are dequantized by the rules of vlo_finalize_weights. */
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

/* Prefill: one stream's n_tokens rows (1 <= n_tokens <= vlo_max_prefill_tokens(e)) through all
 * layers in one pass, with the bits of the same rows fed as vlo_step calls of max_step_tokens (the chunked path).  The
 * layer GEMMs run on gemm_prefill_kernel (tokens on wgmma M, the chunked path's stream-K k-ranges summed in its plane
 * order, csrc/gemm_prefill.cuh); the KV append, fix-up, RMSNorm, lm_head and decision kernels are the step's; each layer's
 * attention is one vlo_step_segments-style launch whose segments are the max_step_tokens pieces, each planned as its own
 * step.  d_row_ids (device int64 [n_tokens] or NULL) as in vlo_step_ids; d_last_logits: bf16 [1, vocab] or NULL;
 * d_decision: one vlo_decision or NULL, at the last row.  vlo_last_step_logits / vlo_last_step_hidden then cover all
 * n_tokens rows.  The stream's pages are taken all or none; on any error the stream is unchanged.  An engine with
 * quantized layer matrices (e4m3 weights, W8A8, int4) prefills only with vlo_set_quantized_prefill: its layer GEMMs then
 * run on gemm_prefill_q_kernel (weights on wgmma M, the chunked kernels' MMAs and partial scaling, csrc/gemm_prefill_q.cuh);
 * without it vlo_prefill returns an error. */
int vlo_prefill(vlo_engine* e, int stream_id, int n_tokens, const int64_t* d_row_ids, const void* d_embeds,
                void* d_last_logits, vlo_decision* d_decision, int interval_id, void* cuda_stream);
/* 8 x max_step_tokens once vlo_finalize_weights has loaded bf16 layer weights, or quantized ones with
 * vlo_set_quantized_prefill: it then grows the token-row workspaces (h, xn, q, attn_out, act, attention workspace, step
 * tables; under FP8 activations also their e4m3 copies and token scales) to that many rows.  0 before, and on engines
 * with quantized layer matrices without vlo_set_quantized_prefill, which keep them at max_step_tokens rows. */
int vlo_max_prefill_tokens(vlo_engine* e);

/* all-position logits for the last vlo_step's tokens (the reference's logits_to_keep=0 behaviour,
 * HF:models/llama/modeling_llama.py:485-487); d_logits bf16 [sum(q_lens), vocab]. Test/compat path.  A quantized lm_head
 * runs in pieces of at most 128 rows; every row's logits are those a step of its own would give. */
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
/* vlo_op_gemm_ws with the token tile chosen by `tiling` when bn <= 0 (0: the smallest covering instance, as
 * vlo_op_gemm_ws; 1: the ViT trunk tiling of 3+ frames; 2: the 64-token fp16 instance that runs beside a decoder step,
 * which is the one vlo_vit_encode uses for 1-2 frames).  h_plan (may be NULL) receives {bn, token tiles, most planes of
 * one tile}.  Asynchronous. */
int vlo_op_gemm_ws_tiled(int fmt, int mode, const void* d_w, int rows_w, const void* d_x, int rows_x, int k, void* d_out,
                         int ld_out, long long plane_stride, const float* d_bias, int act, int n_ctas, int bn, int tiling,
                         int32_t* h_plan, void* cuda_stream);
/* The same GEMM in mode 0 on e4m3 weights (the decoder's FP8 weight form): d_w8 [rows_w, k] e4m3fn bytes, d_scale fp32
 * [rows_w] row scales, X bf16 [rows_x, k].  Same token tile and stream-K plan as the bf16 call with these sizes and
 * n_ctas; each weight k-block is upcast to bf16 exactly and multiplied by the bf16 wgmma chain, so plane p holds
 * fl(P_p[t][n] * d_scale[n]), P_p being plane p of the bf16 call on the upcast weights.  d_out == NULL only plans
 * (*h_max_planes).  Asynchronous. */
int vlo_op_gemm_ws_f8(const void* d_w8, const float* d_scale, int rows_w, const void* d_x, int rows_x, int k, float* d_out,
                      long long plane_stride, int n_ctas, int* h_max_planes, void* cuda_stream);
/* The same GEMM in mode 0 on e4m3 weights AND e4m3 activations (the fp8_activations form): d_w8 / d_scale as above, d_x8
 * [rows_x, k] e4m3fn bytes with fp32 token scales d_xscale [rows_x].  Same token tile and stream-K plan as the bf16
 * call; plane p holds fl(fl(P_p[t][n] * d_scale[n]) * d_xscale[t]), P_p the FP8 wgmma sum of the codes over plane p's
 * k-blocks.  d_out == NULL only plans (*h_max_planes).  Asynchronous. */
int vlo_op_gemm_ws_a8(const void* d_w8, const float* d_scale, int rows_w, const void* d_x8, const float* d_xscale, int rows_x,
                      int k, float* d_out, long long plane_stride, int n_ctas, int* h_max_planes, void* cuda_stream);
/* The same GEMM in mode 0 on int4 weights (the decoder's W4A16 form, see vlo_finalize_weights): d_w4 the codes in the
 * engine byte order, d_gscale bf16 [rows_w, k / 128], X bf16 [rows_x, k], 1 <= rows_x <= 128, k % 128 == 0.  Same token
 * tile and stream-K plan as the bf16 call with these sizes and n_ctas; the codes are dequantized to W4 in registers and
 * multiplied by the bf16 wgmma chain, so every plane is bit for bit that of the bf16 call on W4.  d_out == NULL only
 * plans (*h_max_planes).  Asynchronous. */
int vlo_op_gemm_ws_i4(const void* d_w4, const void* d_gscale, int rows_w, const void* d_x, int rows_x, int k, float* d_out,
                      long long plane_stride, int n_ctas, int* h_max_planes, void* cuda_stream);
/* Whole tiles (mode 1) of e4m3 or int4 weights with the bf16 store: the lm_head of engines with quantized vocabulary
 * matrices.  fmt 2: d_w e4m3 bytes [rows_w, k], d_scale fp32 [rows_w], out = bf16(fl(acc * s[n])), acc the fp32 chain of
 * the bf16 kernel on the upcast codes.  fmt 4: d_w int4 codes in the engine byte order, d_scale bf16 [rows_w, k / 128],
 * k % 128 == 0, rows_x <= 128, out = bf16(acc) = the bf16 whole-tile call on W4.  X bf16 [rows_x, k]; out bf16
 * [rows_x][ld_out].  One CTA covers all of k for each of its tiles, so a row's logits depend on no other row and on no
 * token tile.  n_ctas <= 0: one CTA per SM.  h_plan (optional): {token tile, token tiles, CTAs}.  d_out == NULL only
 * plans.  Asynchronous. */
int vlo_op_gemm_ws_tiles_q(int fmt, const void* d_w, const void* d_scale, int rows_w, const void* d_x, int rows_x, int k,
                           void* d_out, int ld_out, int n_ctas, int32_t* h_plan, void* cuda_stream);
/* The token-embedding gather of vlo_embed_tokens on a bare table: fmt 1 bf16 [vocab, hidden] (d_scale unused), 2 e4m3
 * bytes + fp32 row scales, 4 int4 codes in the engine byte order + bf16 group scales; hidden % 128 == 0.  Row i of
 * d_out (bf16 [n, hidden]) = row min(ids[i], vocab - 1), dequantized; a row with ids[i] < 0 is left alone.
 * Asynchronous. */
int vlo_op_embed_rows_q(int fmt, const void* d_table, const void* d_scale, int vocab, int hidden, const int64_t* d_ids, int n,
                        void* d_out, void* cuda_stream);
/* ViT trunk GEMM (csrc/gemm_vit.cuh), fp16, 128-token x 128-feature tiles:
 * out[t][n] = act(fp16(sum_k X[t,k] W[n,k] + bias[n])), fp16 out[rows_x][ld_out], ld_out even and >= rows_w;
 * n_ctas <= 0: one CTA per SM. */
int vlo_op_gemm_vit(const void* d_w, int rows_w, const void* d_x, int rows_x, int k, void* d_out, int ld_out,
                    const float* d_bias, int act, int n_ctas, void* cuda_stream);
/* KV-append attention over one layer's cache (the graded kernel, K15):
 *   d_q bf16 [n_tok, n_heads, head_dim] (RoPE applied); d_k/d_v bf16 [n_kv_heads, kv_stride, head_dim];
 *   keys 0..kv_len-1 valid, the n_tok query tokens sit at positions kv_len-n_tok .. kv_len-1 (causal with
 *   offset, HF:masking_utils.py:263-272); d_out bf16 [n_tok, n_heads*head_dim]; d_ws fp32 scratch of
 *   vlo_op_attn_ws_bytes(). Replaces HF:models/llama/modeling_llama.py:272-285 (SDPA / flash-attn 2).
 *   Rows kv_len .. kv_stride - 1 are masked and may hold anything, NaN and Inf included.  The n_tok new rows must be
 *   finite: a row multiplies the V rows of the later new tokens of its work item by P = 0 (DESIGN §3). */
int64_t vlo_op_attn_ws_bytes(int n_tok, int n_heads, int head_dim, int kv_len);
int vlo_op_attn_kvappend(const void* d_q, const void* d_k, const void* d_v, void* d_out, float* d_ws, int n_tok,
                         int n_heads, int n_kv_heads, int head_dim, int kv_len, long long kv_stride, void* cuda_stream);
/* kernel-level: the decoder attention over a paged pool [n_pages, n_kv_heads, 64, 128] (tests).  d_page_table: device
 * int32 [ceil(kv_len / 64)], the page of each 64-key block; other arguments as vlo_op_attn_kvappend.  Rows of the last
 * page past kv_len are masked: they may hold anything, NaN and Inf included.  The new rows must be finite, as for
 * vlo_op_attn_kvappend. */
int vlo_op_attn_kvappend_paged(const void* d_q, const void* d_k_pool, const void* d_v_pool, const int32_t* d_page_table,
                               int n_pages, void* d_out, float* d_ws, int n_tok, int n_heads, int n_kv_heads,
                               int head_dim, int kv_len, void* cuda_stream);
/* kernel-level: the attention of one segmented sequence over a paged pool, planned and launched as vlo_step_segments
 * does.  n_tok = sum(h_seg_lens[0..n_segs)) query rows (host array, each > 0) sit at positions kv_len - n_tok ..
 * kv_len - 1 of d_q [n_tok, n_heads, head_dim]; row r attends causally to keys 0..(its position).  Segment j (rows
 * o_j .. o_j + len_j - 1, ending at key e_j = kv_len - n_tok + o_j + len_j) gets in d_out exactly the bits
 * vlo_op_attn_kvappend_paged gives its rows alone with kv_len = e_j on the same pool.  n_segs = 1 is that call.
 * Keys past a row's position are masked.  Rows past kv_len may hold anything, NaN and Inf included; the new rows must
 * be finite, since a row multiplies the V rows of the later tokens of its work item or packed run by P = 0 (DESIGN §3).  Scratch is allocated internally;
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
/* The GEMM configuration vlo_vit_encode runs for n_frames frames of n_patches tokens (rows = n_frames * n_patches),
 * without launching anything: h_out[0..11) =
 *   [0] QKV / fc1 kernel: 0 = vlo_op_gemm_vit, else the vlo_op_gemm_ws_tiled tiling of its mode-1 call
 *   [1] QKV and [2] fc1 token tile;  [3] the vlo_op_gemm_ws_tiled tiling of the out_proj / fc2 mode-0 calls
 *   [4] out_proj token tile and [5] its most planes of one tile;  [6] fc2 token tile and [7] its most planes
 *   [8] the patch-embed and [9] the MAP-head K/V bn of vlo_op_gemm;  [10] the MAP head's token tile (n_frames rows). */
int vlo_op_vit_tiling(int n_frames, int n_patches, int hidden, int mlp, int32_t* h_out);
/* The other kernels of vlo_vit_encode (csrc/vit_kernels.cuh), launched by the same helpers.  Asynchronous.
 * patchify: u8 d_frames [n_frames, 3, S, S] -> fp16 d_out [n_frames * g * g, 3 ps ps] (g = S / ps, ps a multiple of 8),
 *   row b g^2 + py g + px, column (c ps + iy) ps + ix = fp16((x / 255 - 0.5) / 0.5) of pixel (c, py ps + iy, px ps + ix).
 * vit_layernorm: d_in [rows, C] (fp16 if in_is_f16, else fp32) -> LayerNorm with fp32 statistics, affine d_w / d_b, to
 *   d_out16 fp16 and / or d_out32 fp32 (either may be NULL); C <= 12288.
 * vit_fix_ln: d_part fp32 stream-K planes [plane][rows][C] of the fp16 vlo_op_gemm_ws mode-0 call with rows_w = C, this
 *   k, bn and n_ctas (plane_stride rows * C), of which only the planes of each (128-feature, bn-token) tile are read:
 *     h[t][n] = h[t][n] + fp16(sum_s part[s][t][n] + bias[n])   (fp32 residual d_h, summed in plane order)
 *     then LayerNorm(h[t]) -> d_out16 / d_out32 as vit_layernorm.  C a multiple of 4, <= 12288, at most 8 planes;
 *     the fp32 arrays 16-byte and d_out16 8-byte aligned.
 * vit_pool: adaptive average pool of each frame's grid x grid tokens d_in fp32 [n_frames, grid^2, C] to ph x pw cells,
 *   cell i pw + j of frame b -> d_tokens[b n_tok + tok_off + i pw + j] (window rows [i g / ph, ceil((i + 1) g / ph)), cols
 *   alike; summed row by row in fp32, divided once).
 * cls_residual: d_tokens[b n_tok][c] = fp16(d_resid16[b][c] + d_mlp16[b][c]) for the n_frames x C fp16 inputs. */
/* tanh.approx.f32 (the MUFU.TANH the GELU-tanh epilogue evaluates) of n fp32 values: d_y[i] = tanh_approx(d_x[i]).
 * Asynchronous. */
int vlo_op_tanh_approx(const float* d_x, float* d_y, long long n, void* cuda_stream);
int vlo_op_patchify(const uint8_t* d_frames, int n_frames, int image_size, int patch_size, void* d_out, void* cuda_stream);
int vlo_op_vit_layernorm(const void* d_in, int in_is_f16, int rows, int C, const float* d_w, const float* d_b, void* d_out16,
                         float* d_out32, float eps, void* cuda_stream);
int vlo_op_vit_fix_ln(const float* d_part, int rows, int C, int k, int bn, int n_ctas, const float* d_bias, float* d_h,
                      const float* d_ln_w, const float* d_ln_b, void* d_out16, float* d_out32, float eps, void* cuda_stream);
int vlo_op_vit_pool(const float* d_in, int n_frames, int grid, int C, int ph, int pw, int n_tok, int tok_off, float* d_tokens,
                    void* cuda_stream);
int vlo_op_cls_residual(const void* d_resid16, const void* d_mlp16, float* d_tokens, int n_frames, int C, int n_tok,
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
/* vlo_op_resid_rmsnorm that also writes the e4m3 row d_xq [T, H] of each bf16 xn row and its fp32 scale d_xs [T], by
 * the rule of vlo_set_fp8_activations; d_xn (not NULL here) gets the same bits as from vlo_op_resid_rmsnorm.
 * Asynchronous. */
int vlo_op_resid_rmsnorm_q8(const float* d_part, int k, int n_ctas, void* d_h, const void* d_w, void* d_xn, void* d_xn_last,
                            const int32_t* d_last_index, void* d_xq, float* d_xs, int T, int H, float eps, void* cuda_stream);
/* The per-token e4m3 quantizer of the attention output and of act: bf16 d_x [T, K] (K a multiple of 8) -> e4m3fn
 * d_q [T, K] and fp32 d_s [T], by the rule of vlo_set_fp8_activations.  Asynchronous. */
int vlo_op_quant_rows_e4m3(const void* d_x, int T, int K, void* d_q, float* d_s, void* cuda_stream);
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
/* Prefill GEMM (csrc/gemm_prefill.cuh), bf16 W [rows_w, k], X [rows_x, k] (any rows_x): for each output the k-ranges of
 * the stream-K plan vlo_op_gemm_ws (mode 0, one token tile) makes over n_ctas CTAs (0: all SMs), each an in-order chain
 * from zero, summed in plane order.  epi 0: d_out fp32 [rows_x, rows_w] = 0 + P0 + P1 + ..., what the fix-up kernels sum
 * from the chunked path's planes; epi 1: d_out bf16 [rows_x, rows_w / 2], the SwiGLU of vlo_op_gemm_swiglu's tile layout
 * (rows_w % 128 == 0, all SMs' plan) on g, u = P0 + P1 + ....  Rows past rows_x are not written.  Asynchronous. */
int vlo_op_gemm_prefill(int epi, const void* d_w, int rows_w, const void* d_x, int rows_x, int k, int n_ctas, void* d_out,
                        void* cuda_stream);
/* Prefill GEMM of quantized weights (csrc/gemm_prefill_q.cuh), with the operands of vlo_op_gemm_ws_f8 (fmt 2: d_w e4m3
 * [rows_w, k], d_scale fp32 [rows_w]), vlo_op_gemm_ws_a8 (fmt 3: the same weights, d_x e4m3 [rows_x, k] with fp32 token
 * scales d_xscale [rows_x]) or vlo_op_gemm_ws_i4 (fmt 4: d_w the codes, d_gscale bf16 [rows_w, k / 128]); the unused
 * pointers may be NULL.  Any rows_x; plan and epilogues as vlo_op_gemm_prefill, with each range's partial scaled as the
 * chunked kernels scale a partial before it is summed (fmt 2: fl(P * d_scale[n]); fmt 3: fl(fl(P * d_scale[n]) *
 * d_xscale[t]); fmt 4: P).  So epi 0 equals vlo_op_gemm_ws_{f8,a8,i4} mode 0 on each 128-row chunk of X summed
 * 0 + plane 0 + plane 1 + ..., and epi 1 equals vlo_op_gemm_swiglu_{f8,a8,i4} on each chunk.  Asynchronous. */
int vlo_op_gemm_prefill_q(int fmt, int epi, const void* d_w, const float* d_scale, const void* d_gscale, int rows_w,
                          const void* d_x, const float* d_xscale, int rows_x, int k, int n_ctas, void* d_out,
                          void* cuda_stream);
/* vlo_op_gemm_swiglu on e4m3 weights d_w8 [rows_w, k] with fp32 row scales d_scale [rows_w] (same row order and plan):
 * g, u = bf16(sum_p fl(P_p * d_scale[n])) summed in plane order, P_p the fp32 partials of the bf16 kernel on the exactly
 * upcast weights (the finisher's own partial is plane 0).  Asynchronous. */
int vlo_op_gemm_swiglu_f8(const void* d_w8, const float* d_scale, int rows_w, const void* d_x, int rows_x, int k, void* d_act,
                          float* d_planes, int64_t plane_elems, int32_t* d_flags, int n_flags, void* cuda_stream);
/* vlo_op_gemm_swiglu on e4m3 weights (d_w8, d_scale) and e4m3 activations d_x8 [rows_x, k] with fp32 token scales
 * d_xscale: g, u = bf16(sum_p fl(fl(P_p * d_scale[n]) * d_xscale[t])) in plane order, P_p the FP8 wgmma partials (the
 * finisher's own partial is plane 0).  Asynchronous. */
int vlo_op_gemm_swiglu_a8(const void* d_w8, const float* d_scale, int rows_w, const void* d_x8, const float* d_xscale,
                          int rows_x, int k, void* d_act, float* d_planes, int64_t plane_elems, int32_t* d_flags, int n_flags,
                          void* cuda_stream);
/* vlo_op_gemm_swiglu on int4 weights (d_w4, d_gscale as in vlo_op_gemm_ws_i4; same row order and plan): bit for bit
 * vlo_op_gemm_swiglu on W4.  Asynchronous. */
int vlo_op_gemm_swiglu_i4(const void* d_w4, const void* d_gscale, int rows_w, const void* d_x, int rows_x, int k, void* d_act,
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

/* Test hooks for the PDL contract (csrc/ptx.cuh): before its grid dependency resolves, a kernel reads nothing an
 * earlier kernel of the step writes and writes nothing to global memory.
 * vlo_op_pdl_arm arms a one-shot probe.  Every vlo_op_* entry above that launches a PDL kernel, and vlo_letterbox /
 * vlo_letterbox_planes, launch the armed probe on their stream right before their first PDL launch (after their own
 * table uploads) and disarm it.  The probe kernel runs on a few CTAs, lets its dependents launch at once, spins on the
 * global timer for spin_ns (0 < spin_ns <= 2 ms), then copies n_chunks chunks of `bytes` bytes, chunk i at byte offset
 * i * chunk_stride of both pointers: mode VLO_PDL_LATE_WRITE src -> dst (the operand arrives after the kernel under test
 * has started); VLO_PDL_LATE_READ exchanges them: src receives a snapshot of what that kernel had written to dst by
 * then, dst what src held (so a region can hold a marker before the launch and the values the kernel expects after
 * its wait, e.g. zero arrival counters).  Ranges must not overlap.  vlo_op_pdl_probe_count: probes that ran to completion (synchronises the device); -1 on error. */
enum { VLO_PDL_LATE_WRITE = 1, VLO_PDL_LATE_READ = 2 };
int vlo_op_pdl_arm(int mode, void* d_dst, void* d_src, long long bytes, int n_chunks, long long chunk_stride,
                   long long spin_ns);
long long vlo_op_pdl_probe_count(void);
/* A PDL canary through the product's launch helper: n_words 32-bit words d_src -> d_dst.  variant 0 waits for the grid
 * dependency, then copies; 1 reads d_src before the wait (a read violation); 2 writes d_dst before the wait (a write
 * violation).  Asynchronous. */
int vlo_op_pdl_canary(int variant, const void* d_src, void* d_dst, int n_words, void* cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* VLO_B200_H_ */
