// Host side of the KV-append attention: chunking of sequences into <=64-row work items,
// split-KV planning (one wave of CTAs over the SMs), workspace layout and launches.
// The plan depends only on (q_len, kv_len) of the sequences, so a decoder step builds and
// uploads it once and reuses it for all layers.
#include "attn.cuh"

#include <algorithm>
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
// work items of any plan over total_tokens rows: every sequence or segment holds at least one token
int max_items(int total_tokens, int G) { return max_chunks(total_tokens, total_tokens, G); }
// Items of single-segment sequences: n_splits <= max(1, n_sms / (n_kv_heads * n_items)) and rows <= 64, so the sum of
// n_kv_heads * n_splits * rows over them is bounded by (n_sms + n_kv_heads * n_items) * 64.  A segment of a segmented
// sequence is planned as if alone: each of its items has n_kv_heads * n_splits <= max(n_kv_heads, n_sms) and q_count * G
// rows, so all segments together stay below (n_sms + n_kv_heads) * G * total_tokens.
size_t cap_slots_for(int total_tokens, int n_seqs, int n_heads, int n_kv_heads) {
  const int G = n_heads / n_kv_heads;
  return static_cast<size_t>(num_sms() + n_kv_heads * max_chunks(total_tokens, n_seqs, G)) * 128 +
         static_cast<size_t>(num_sms() + n_kv_heads) * G * total_tokens;
}
}  // namespace

// The item table is bounded by max_items (one segment per token at most), which holds for any number of sequences, so
// the staging does not depend on n_seqs (kept for symmetry with attn_ws_bytes, whose split-KV slots do).
size_t attn_stage_bytes(int total_tokens, int n_seqs, int n_heads, int n_kv_heads) {
  (void)n_seqs;
  const int G = n_heads / n_kv_heads;
  return align256(sizeof(AttnItem) * max_items(total_tokens, G)) + align256(sizeof(int) * total_tokens) +
         align256(sizeof(AttnCluster) * max_items(total_tokens, G)) + align256(sizeof(AttnPack) * max_items(total_tokens, G));
}

size_t attn_ws_bytes(int total_tokens, int n_seqs, int n_heads, int n_kv_heads) {
  const int G = n_heads / n_kv_heads;
  const size_t slots = cap_slots_for(total_tokens, n_seqs, n_heads, n_kv_heads);
  return align256(slots * kAttnHD * 4) + align256(slots * 2 * 4) +
         align256(sizeof(AttnItem) * max_items(total_tokens, G)) + align256(sizeof(int) * total_tokens) +
         align256(sizeof(AttnCluster) * max_items(total_tokens, G)) + align256(sizeof(AttnPack) * max_items(total_tokens, G));
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
  std::vector<int> item_want;  // split budget of each item; 0 = the budget shared by single-segment sequences
  std::vector<int> item_seq;   // segmented sequence of each item, -1 for a single-segment sequence
  std::vector<char> item_one;  // the item is a one-token segment of a segmented sequence
  std::vector<int> tok_item(total_tokens, 0);
  // rows [q_tok0, q_tok0 + q_len) at positions kv_end - q_len .. kv_end - 1, chunked from the first row
  auto chunk = [&](int q_tok0, int q_len, int kv_end, int pt0, int want, int seq) {
    for (int t0 = 0; t0 < q_len; t0 += per) {
      AttnItem it{};
      it.q_tok0 = q_tok0 + t0;
      it.q_count = std::min(per, q_len - t0);
      it.q_pos0 = kv_end - q_len + t0;
      it.pt0 = pt0;
      for (int t = 0; t < it.q_count; ++t) tok_item[it.q_tok0 + t] = static_cast<int>(items.size());
      items.push_back(it);
      item_want.push_back(want);
      item_seq.push_back(seq);
      item_one.push_back(seq >= 0 && q_len == 1);
    }
  };
  int n_shared = 0;
  for (int s = 0; s < n_seqs; ++s) {
    const AttnSeq& q = seqs[s];
    VLO_CHECK(q.q_len > 0 && q.kv_len >= q.q_len, "bad sequence lengths");
    VLO_CHECK(q.pt0 >= 0, "page-table offset out of range");
    if (q.n_segs <= 1) {
      chunk(q.q_tok0, q.q_len, q.kv_len, q.pt0, 0, -1);
      n_shared += (q.q_len + per - 1) / per;
      continue;
    }
    // Each segment gets the items, split budget and split grid a one-sequence step of that segment alone gets: its
    // rows are then computed with the same partials and the same merge.  Keys of later segments lie past every row's
    // causal limit and are masked like the stale rows of a last page.
    int off = 0;
    for (int j = 0; j < q.n_segs; ++j) {
      const int len = q.seg_lens[j];
      VLO_CHECK(len > 0, "segment lengths must be positive");
      off += len;
      VLO_CHECK(off <= q.q_len, "segment lengths exceed the sequence's q_len");
      const int seg_items = (len + per - 1) / per;
      chunk(q.q_tok0 + off - len, len, q.kv_len - q.q_len + off, q.pt0,
            std::max(1, num_sms() / (n_kv_heads * seg_items)), s);
    }
    VLO_CHECK(off == q.q_len, "segment lengths must add up to the sequence's q_len");
  }
  const int n_items = static_cast<int>(items.size());
  const int want_shared = std::max(1, num_sms() / (n_kv_heads * std::max(1, n_shared)));
  int max_splits = 1, max_bps = 2;
  size_t slots = 0;
  double algo = 0.0;
  for (const AttnItem& it : items)  // SURVEY 8(d): K+V rows read once per item, Q read, output written
    algo += static_cast<double>(it.q_pos0 + it.q_count) * n_kv_heads * kAttnHD * 2 * 2 +
            static_cast<double>(it.q_count) * n_heads * kAttnHD * 2 * 2;
  plan->algo_bytes = algo;
  for (size_t i = 0; i < items.size(); ++i) {
    AttnItem& it = items[i];
    const int want = item_want[i] ? item_want[i] : want_shared;
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
  VLO_CHECK(n_items <= max_items(total_tokens, G), "too many attention work items");

  // Packs: runs of 2 .. per consecutive one-token segments of a sequence whose solo items share the split grid (a run
  // is cut where n_splits or blocks_per_split change) go to attn_kvappend_packed_kernel, one CTA per (split, kv head)
  // for the whole run.  Packed items move behind all others, in order.
  std::vector<AttnPack> packs;
  std::vector<int> in_pack(n_items, 0);
  for (int i = 0; i < n_items;) {
    int j = i + 1;
    if (item_one[i])
      while (j < n_items && j - i < per && item_one[j] && item_seq[j] == item_seq[i] &&
             items[j].n_splits == items[i].n_splits && items[j].blocks_per_split == items[i].blocks_per_split)
        ++j;
    if (j - i >= 2) {
      packs.push_back(AttnPack{i, j - i});
      for (int k = i; k < j; ++k) in_pack[k] = 1;
    }
    i = j;
  }

  // Clusters: the items of one segmented sequence with the same blocks_per_split read the same key blocks of the same
  // pages, so attn_kvappend_cluster_kernel loads each block once for up to kAttnClusterMax of them.  Clustered items
  // move behind the others (the item order changes no result); groups of one stay with attn_kvappend_kernel.
  std::vector<std::vector<int>> groups;
  for (int s = 0; s < n_seqs; ++s) {
    std::vector<std::pair<int, std::vector<int>>> by_bps;
    for (int i = 0; i < n_items; ++i) {
      if (item_seq[i] != s || in_pack[i]) continue;
      auto g = std::find_if(by_bps.begin(), by_bps.end(), [&](const auto& x) { return x.first == items[i].blocks_per_split; });
      if (g == by_bps.end()) by_bps.push_back({items[i].blocks_per_split, {i}});
      else g->second.push_back(i);
    }
    for (auto& g : by_bps)
      if (g.second.size() >= 2) groups.push_back(g.second);
  }
  // Clusters of 2: on an H100 at 12k / 66k keys larger clusters measured slower than one CTA per item (the whole
  // cluster advances at the pace of its slowest CTA's ring release), pairs faster (DESIGN.md section 5).
  const int cs = 2;
  std::vector<int> order, in_cluster(n_items, 0);
  std::vector<AttnCluster> clusters;
  for (const auto& g : groups) {
    const int n = static_cast<int>(g.size()), k = (n + cs - 1) / cs;
    for (int c = 0; c < k; ++c) {  // member r of cluster c: item g[c + r * k] (round robin keeps the clusters even)
      AttnCluster cl;
      for (int r = 0; r < kAttnClusterMax; ++r) cl.item[r] = -1;
      for (int r = 0, j = c; j < n; ++r, j += k) cl.item[r] = g[j];
      clusters.push_back(cl);
    }
    for (int i : g) in_cluster[i] = 1;
  }
  for (int i = 0; i < n_items; ++i)
    if (!in_cluster[i] && !in_pack[i]) order.push_back(i);
  const int n_plain = static_cast<int>(order.size());
  int max_cluster_splits = 1, max_pack_splits = 1;
  for (int i = 0; i < n_items; ++i)
    if (in_cluster[i]) {
      order.push_back(i);
      max_cluster_splits = std::max(max_cluster_splits, items[i].n_splits);
    }
  for (int i = 0; i < n_items; ++i)
    if (in_pack[i]) {
      order.push_back(i);
      max_pack_splits = std::max(max_pack_splits, items[i].n_splits);
    }
  if (!clusters.empty() || !packs.empty()) {
    std::vector<int> pos(n_items);
    std::vector<AttnItem> reordered(n_items);
    for (int j = 0; j < n_items; ++j) {
      pos[order[j]] = j;
      reordered[j] = items[order[j]];
    }
    items.swap(reordered);
    for (int& t : tok_item) t = pos[t];
    for (AttnCluster& cl : clusters)
      for (int r = 0; r < kAttnClusterMax; ++r)
        if (cl.item[r] >= 0) cl.item[r] = pos[cl.item[r]];
    for (AttnPack& pk : packs) pk.item0 = pos[pk.item0];  // a run's items stay consecutive and in order
  }
  plan->n_plain = n_plain;
  plan->n_clusters = static_cast<int>(clusters.size());
  plan->cluster_size = cs;
  plan->max_cluster_splits = max_cluster_splits;
  plan->n_packs = static_cast<int>(packs.size());
  plan->n_packed_items = static_cast<int>(std::count(in_pack.begin(), in_pack.end(), 1));
  plan->max_pack_splits = max_pack_splits;
  plan->n_items = n_items;
  plan->max_splits = max_splits;
  plan->max_blocks_per_split = max_bps;
  plan->total_tokens = total_tokens;
  if (d_ws == nullptr) return 0;

  // workspace carve-up (same order as attn_ws_bytes)
  uint8_t* w = static_cast<uint8_t*>(d_ws);
  plan->ws_o = reinterpret_cast<float*>(w);
  w += align256(cap_slots * kAttnHD * 4);
  plan->ws_ml = reinterpret_cast<float*>(w);
  w += align256(cap_slots * 2 * 4);
  plan->d_items = w;
  w += align256(sizeof(AttnItem) * max_items(total_tokens, G));
  plan->d_tok_item = reinterpret_cast<int*>(w);
  w += align256(sizeof(int) * total_tokens);
  plan->d_clusters = w;
  w += align256(sizeof(AttnCluster) * max_items(total_tokens, G));
  plan->d_packs = w;

  uint8_t* hs = static_cast<uint8_t*>(h_stage);
  std::memcpy(hs, items.data(), sizeof(AttnItem) * n_items);
  uint8_t* hs2 = hs + align256(sizeof(AttnItem) * max_items(total_tokens, G));
  std::memcpy(hs2, tok_item.data(), sizeof(int) * total_tokens);
  VLO_CUDA(cudaMemcpyAsync(plan->d_items, hs, sizeof(AttnItem) * n_items, cudaMemcpyHostToDevice, stream));
  VLO_CUDA(cudaMemcpyAsync(plan->d_tok_item, hs2, sizeof(int) * total_tokens, cudaMemcpyHostToDevice, stream));
  uint8_t* hs3 = hs2 + align256(sizeof(int) * total_tokens);
  if (!clusters.empty()) {
    std::memcpy(hs3, clusters.data(), sizeof(AttnCluster) * clusters.size());
    VLO_CUDA(cudaMemcpyAsync(plan->d_clusters, hs3, sizeof(AttnCluster) * clusters.size(), cudaMemcpyHostToDevice, stream));
  }
  if (!packs.empty()) {
    uint8_t* hs4 = hs3 + align256(sizeof(AttnCluster) * max_items(total_tokens, G));
    std::memcpy(hs4, packs.data(), sizeof(AttnPack) * packs.size());
    VLO_CUDA(cudaMemcpyAsync(plan->d_packs, hs4, sizeof(AttnPack) * packs.size(), cudaMemcpyHostToDevice, stream));
  }
  return 0;
}

// A cluster of cs attention CTAs (one SM each) can be resident: cudaOccupancyMaxActiveClusters, once per (cs, smem).
static bool cluster_launch_fits(int cs, size_t smem) {
  static int known[kAttnClusterMax + 1] = {};  // 0 unknown, 1 fits, -1 does not
  static size_t known_smem[kAttnClusterMax + 1] = {};
  if (known[cs] != 0 && known_smem[cs] == smem) return known[cs] > 0;
  if (ensure_max_smem(reinterpret_cast<const void*>(attn_kvappend_cluster_kernel), kAttnSmemOptIn)) return false;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(cs, 1, 1);
  cfg.blockDim = dim3(kAttnThreads);
  cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cs;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, attn_kvappend_cluster_kernel, &cfg) != cudaSuccess) {
    cudaGetLastError();
    n = 0;
  }
  known[cs] = n > 0 ? 1 : -1;
  known_smem[cs] = smem;
  return n > 0;
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
  const size_t smem = attn_smem_bytes(plan.max_blocks_per_split);
  const bool clustered = plan.n_clusters > 0 && cluster_launch_fits(plan.cluster_size, smem);
  // without clusters every item but the packed ones runs alone
  const int n_plain = clustered ? plan.n_plain : plan.n_items - plan.n_packed_items;
  prof_begin(PROF_ATTN, stream, plan.algo_bytes);
  if (n_plain > 0) {
    VLO_CUDA(launch_pdl(attn_kvappend_kernel, dim3(plan.max_splits, n_kv_heads, n_plain), dim3(kAttnThreads), smem, stream,
                        tk, tv, p));
    count_launch();
  }
  if (clustered) {
    if (ensure_max_smem(reinterpret_cast<const void*>(attn_kvappend_cluster_kernel), kAttnSmemOptIn)) return -1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(plan.cluster_size * plan.n_clusters, plan.max_cluster_splits, n_kv_heads);
    cfg.blockDim = dim3(kAttnThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = plan.cluster_size;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 2 : 1;
    VLO_CUDA(cudaLaunchKernelEx(&cfg, attn_kvappend_cluster_kernel, tk, tv, p,
                                static_cast<const AttnCluster*>(plan.d_clusters)));
    count_launch();
  }
  if (plan.n_packs > 0) {
    if (ensure_max_smem(reinterpret_cast<const void*>(attn_kvappend_packed_kernel), kAttnSmemOptIn)) return -1;
    VLO_CUDA(launch_pdl(attn_kvappend_packed_kernel, dim3(plan.max_pack_splits, n_kv_heads, plan.n_packs),
                        dim3(kAttnThreads), smem, stream, tk, tv, p, static_cast<const AttnPack*>(plan.d_packs)));
    count_launch();
  }
  prof_end(stream);
  if (plan.skip_merge) return 0;
  return launch_merge(plan, d_out, n_heads, n_kv_heads, scale_log2, stream);
}

}  // namespace vlo
