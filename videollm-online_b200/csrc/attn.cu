// Host side of the KV-append attention: chunking of sequences into <=64-row work items,
// split-KV planning (one wave of CTAs over the SMs), workspace layout and launches.
// The plan depends only on (q_len, kv_len) of the sequences, so a decoder step builds and
// uploads it once and reuses it for all layers.
#include "attn.cuh"

#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "common.h"
#include "kv_pages.h"

namespace vlo {

// every 64-key TMA box of the attention lies in one page of the KV pool
static_assert(kKvPageTokens == kAttnBlk, "KV page size must equal the attention key block");

namespace {
int max_chunks(int total_tokens, int n_seqs, int G) {
  const int per = std::max(1, 64 / G);
  return total_tokens / per + n_seqs + 1;
}
// Per item n_splits <= max(1, n_sms / (n_kv_heads * n_items)) and rows <= 64, so the sum of
// n_kv_heads * n_splits * rows over all items is bounded by (n_sms + n_kv_heads * n_items) * 64.
size_t cap_slots_for(int total_tokens, int n_seqs, int n_heads, int n_kv_heads) {
  const int G = n_heads / n_kv_heads;
  return static_cast<size_t>(num_sms() + n_kv_heads * max_chunks(total_tokens, n_seqs, G)) * 128;
}
}  // namespace

size_t attn_stage_bytes(int total_tokens, int n_seqs, int n_heads, int n_kv_heads) {
  const int G = n_heads / n_kv_heads;
  return align256(sizeof(AttnItem) * max_chunks(total_tokens, n_seqs, G)) + align256(sizeof(int) * total_tokens);
}

size_t attn_ws_bytes(int total_tokens, int n_seqs, int n_heads, int n_kv_heads) {
  const int G = n_heads / n_kv_heads;
  const size_t slots = cap_slots_for(total_tokens, n_seqs, n_heads, n_kv_heads);
  return align256(slots * kAttnHD * 4) + align256(slots * 2 * 4) +
         align256(sizeof(AttnItem) * max_chunks(total_tokens, n_seqs, G)) + align256(sizeof(int) * total_tokens);
}

int attn_plan(AttnPlan* plan, void* d_ws, void* h_stage, const AttnSeq* seqs, int n_seqs, int total_tokens,
              int n_heads, int n_kv_heads, int head_dim, cudaStream_t stream) {
  VLO_CHECK(head_dim == kAttnHD, "decoder attention kernel is built for head_dim 128");
  VLO_CHECK(n_heads % n_kv_heads == 0, "n_heads must be a multiple of n_kv_heads");
  const int G = n_heads / n_kv_heads;
  VLO_CHECK(G <= 64, "GQA group too large");
  const int per = 64 / G;        // query tokens per work item
  const int blk = kAttnBlk;      // keys per pipeline block
  plan->blk = blk;

  std::vector<AttnItem> items;
  std::vector<int> tok_item(total_tokens, 0);
  for (int s = 0; s < n_seqs; ++s) {
    const AttnSeq& q = seqs[s];
    VLO_CHECK(q.q_len > 0 && q.kv_len >= q.q_len, "bad sequence lengths");
    VLO_CHECK(q.pt0 >= 0, "page-table offset out of range");
    for (int t0 = 0; t0 < q.q_len; t0 += per) {
      AttnItem it{};
      it.q_tok0 = q.q_tok0 + t0;
      it.q_count = std::min(per, q.q_len - t0);
      it.q_pos0 = q.kv_len - q.q_len + t0;
      it.pt0 = q.pt0;
      for (int t = 0; t < it.q_count; ++t) tok_item[it.q_tok0 + t] = static_cast<int>(items.size());
      items.push_back(it);
    }
  }
  const int n_items = static_cast<int>(items.size());
  const int want = std::max(1, num_sms() / (n_kv_heads * n_items));
  int max_splits = 1, max_bps = 2;
  size_t slots = 0;
  double algo = 0.0;
  for (const AttnItem& it : items)  // SURVEY 8(d): K+V rows read once per item, Q read, output written
    algo += static_cast<double>(it.q_pos0 + it.q_count) * n_kv_heads * kAttnHD * 2 * 2 +
            static_cast<double>(it.q_count) * n_heads * kAttnHD * 2 * 2;
  plan->algo_bytes = algo;
  for (AttnItem& it : items) {
    const int nblk = (it.q_pos0 + it.q_count + blk - 1) / blk;
    int bps = (nblk + want - 1) / want;
    bps = std::max(2, bps + (bps & 1));  // even: both warp groups get the same number of blocks
    it.blocks_per_split = bps;
    VLO_CHECK(bps <= kAttnPtMax, "attention split of " + std::to_string(bps) + " key blocks exceeds the " +
                                   std::to_string(kAttnPtMax) + " page-table entries a CTA can stage");
    max_bps = std::max(max_bps, bps);
    it.n_splits = (nblk + bps - 1) / bps;
    it.ws_slot0 = static_cast<int>(slots);
    slots += static_cast<size_t>(n_kv_heads) * it.n_splits * it.q_count * G;
    max_splits = std::max(max_splits, it.n_splits);
  }
  const size_t cap_slots = cap_slots_for(total_tokens, n_seqs, n_heads, n_kv_heads);
  VLO_CHECK(slots <= cap_slots, "attention workspace plan overflow");
  VLO_CHECK(n_items <= max_chunks(total_tokens, n_seqs, G), "too many attention work items");

  // workspace carve-up (same order as attn_ws_bytes)
  uint8_t* w = static_cast<uint8_t*>(d_ws);
  plan->ws_o = reinterpret_cast<float*>(w);
  w += align256(cap_slots * kAttnHD * 4);
  plan->ws_ml = reinterpret_cast<float*>(w);
  w += align256(cap_slots * 2 * 4);
  plan->d_items = w;
  w += align256(sizeof(AttnItem) * max_chunks(total_tokens, n_seqs, G));
  plan->d_tok_item = reinterpret_cast<int*>(w);
  plan->n_items = n_items;
  plan->max_splits = max_splits;
  plan->max_blocks_per_split = max_bps;
  plan->total_tokens = total_tokens;

  uint8_t* hs = static_cast<uint8_t*>(h_stage);
  std::memcpy(hs, items.data(), sizeof(AttnItem) * n_items);
  uint8_t* hs2 = hs + align256(sizeof(AttnItem) * max_chunks(total_tokens, n_seqs, G));
  std::memcpy(hs2, tok_item.data(), sizeof(int) * total_tokens);
  VLO_CUDA(cudaMemcpyAsync(plan->d_items, hs, sizeof(AttnItem) * n_items, cudaMemcpyHostToDevice, stream));
  VLO_CUDA(cudaMemcpyAsync(plan->d_tok_item, hs2, sizeof(int) * total_tokens, cudaMemcpyHostToDevice, stream));
  return 0;
}

int attn_max_key_blocks() { return kAttnPtMax - 1; }  // blocks_per_split rounds an odd block count up by one

static int launch_merge(const AttnPlan& plan, void* d_out, int n_heads, int n_kv_heads, float scale_log2, cudaStream_t stream) {
  AttnMergeParams mp{};
  mp.ws_o = plan.ws_o;
  mp.ws_ml = plan.ws_ml;
  mp.items = static_cast<const AttnItem*>(plan.d_items);
  mp.tok_item = plan.d_tok_item;
  mp.out = static_cast<__nv_bfloat16*>(d_out);
  mp.n_heads = n_heads;
  mp.n_kv_heads = n_kv_heads;
  mp.scale_log2 = scale_log2;
  prof_begin(PROF_ATTN_MERGE, stream, 0.0);
  VLO_CUDA(launch_pdl(attn_merge_kernel, dim3(n_heads, plan.total_tokens), dim3(128), 0, stream, mp));
  prof_end(stream);
  count_launch();
  return 0;
}

int attn_run(const AttnPlan& plan, const void* d_q, const void* d_k, const void* d_v, long long kv_rows,
             const int* d_page_table, long long page_stride_rows, long long head_stride_rows, void* d_out, int n_heads,
             int n_kv_heads, int head_dim, cudaStream_t stream) {
  VLO_CHECK(kv_rows > 0 && kv_rows < (1ll << 31), "KV matrix rows out of range for a TMA map");
  VLO_CHECK(page_stride_rows > 0 && page_stride_rows < (1ll << 31) && head_stride_rows >= 0 && head_stride_rows < (1ll << 31),
            "KV page strides out of range");
  CUtensorMap tk, tv;
  if (tmap_2d_sw128(d_k, static_cast<int>(kv_rows), kAttnHD, kAttnBlk, 1, &tk) != 0) return -1;
  if (tmap_2d_sw128(d_v, static_cast<int>(kv_rows), kAttnHD, kAttnBlk, 1, &tv) != 0) return -1;
  if (ensure_max_smem(reinterpret_cast<const void*>(attn_kvappend_kernel), kAttnSmemOptIn)) return -1;
  const float scale_log2 = static_cast<float>(1.4426950408889634 / std::sqrt(static_cast<double>(head_dim)));
  AttnParams p{};
  p.q = static_cast<const __nv_bfloat16*>(d_q);
  p.ws_o = plan.ws_o;
  p.ws_ml = plan.ws_ml;
  p.items = static_cast<const AttnItem*>(plan.d_items);
  p.page_table = d_page_table;
  p.page_stride_rows = static_cast<int>(page_stride_rows);
  p.head_stride_rows = static_cast<int>(head_stride_rows);
  p.n_heads = n_heads;
  p.n_kv_heads = n_kv_heads;
  p.scale_log2 = scale_log2;
  prof_begin(PROF_ATTN, stream, plan.algo_bytes);
  VLO_CUDA(launch_pdl(attn_kvappend_kernel, dim3(plan.max_splits, n_kv_heads, plan.n_items), dim3(kAttnThreads),
                      attn_smem_bytes(plan.max_blocks_per_split), stream, tk, tv, p));
  prof_end(stream);
  count_launch();
  if (plan.skip_merge) return 0;
  return launch_merge(plan, d_out, n_heads, n_kv_heads, scale_log2, stream);
}

}  // namespace vlo
