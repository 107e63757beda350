// KV-cache page pool: the one place that decides where a stream's cache position lives.
//
// Device layout, per layer and K / V: [page][kv_head][kKvPageTokens][128] bf16.  A page holds 64 cache positions of
// every kv head; page p has the same index in every layer, so one page table per stream serves all layers.  Rows are
// counted in units of head_dim (128) elements, as the TMA maps and the append kernel address them.
//
// The host owns the free list and the page tables.  A page handed out may hold stale rows from an earlier owner; they
// are finite (the pool is zero-filled once, and only finite K / V rows are ever written), which is what a masked key of
// the attention needs (it contributes 0 x V).  A host image of a stream (vlo_kv_swap_out / vlo_kv_swap_in) moves
// whole pages, so a swapped-in last page carries the rows past kv_len that it had in the pool: finite as well.
#pragma once
#include <algorithm>
#include <string>
#include <vector>

#include "common.h"

namespace vlo {

constexpr int kKvPageTokens = 64;

inline int kv_pages_for(long long tokens) { return static_cast<int>((tokens + kKvPageTokens - 1) / kKvPageTokens); }

struct KvPool {
  int n_kv_heads = 0;
  int n_pages = 0;
  std::vector<int> free_list;             // stack: back() is handed out next, released pages go back on top
  std::vector<std::vector<int>> tables;   // per stream slot: entry j = page of cache positions [64 j, 64 j + 64)

  void init(int n_streams, int kv_heads, int pages) {
    n_kv_heads = kv_heads;
    n_pages = pages;
    free_list.clear();
    for (int p = pages - 1; p >= 0; --p) free_list.push_back(p);  // page 0 first
    tables.assign(n_streams, {});
  }
  // rows between consecutive pages / kv heads in one layer's K or V matrix
  long long page_stride_rows() const { return static_cast<long long>(n_kv_heads) * kKvPageTokens; }
  static constexpr int head_stride_rows() { return kKvPageTokens; }
  long long rows_per_layer() const { return static_cast<long long>(n_pages) * page_stride_rows(); }
  // row of (cache position pos, kv head 0) of stream sid
  long long row(int sid, int pos) const {
    return tables[sid][pos / kKvPageTokens] * page_stride_rows() + pos % kKvPageTokens;
  }
  int free_pages() const { return static_cast<int>(free_list.size()); }
  // pages stream sid still lacks to hold len positions
  int missing(int sid, int len) const { return std::max(0, kv_pages_for(len) - static_cast<int>(tables[sid].size())); }
  // Size stream sid's table to exactly ceil(len / 64) pages.  Fails without changing anything if the pool is short.
  int resize(int sid, int len) {
    const int need = missing(sid, len);
    if (need > free_pages())
      return fail("KV page pool exhausted: " + std::to_string(need) + " more pages of " + std::to_string(kKvPageTokens) +
                  " tokens needed, " + std::to_string(free_pages()) + " of " + std::to_string(n_pages) + " free");
    std::vector<int>& t = tables[sid];
    const size_t want = static_cast<size_t>(kv_pages_for(len));
    while (t.size() > want) {
      free_list.push_back(t.back());
      t.pop_back();
    }
    while (t.size() < want) {
      t.push_back(free_list.back());
      free_list.pop_back();
    }
    return 0;
  }
};

}  // namespace vlo
