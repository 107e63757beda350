// KV-cache page pool: the one owner of a stream slot's cache state (open or not, length, page table), of the free list
// and of the swap-out gates.
//
// Device layout, per layer and K / V: [page][kv_head][kKvPageTokens][128] bf16.  A page holds 64 cache positions of
// every kv head; page p has the same index in every layer, so one page table per stream serves all layers.  Rows are
// counted in units of head_dim (128) elements, as the TMA maps and the append kernel address them.
//
// Between calls a stream holds exactly ceil(len / 64) pages.  A call that adds rows takes the pages (grow), enqueues
// the work that writes them, then sets the length (commit); a call that fails first gives the pages back (rollback).
//
// A page handed out may hold stale rows from an earlier owner, and a stream's last page keeps whatever its rows past
// kv_len held before a truncate, evict or compact.  Masked rows may hold anything, NaN and Inf included: the attention
// masks their scores and zeroes their V rows in the shared-memory stage (csrc/attn.cuh).  A host image of a stream
// (vlo_kv_swap_out / vlo_kv_swap_in) moves whole pages, so a swapped-in last page carries the rows past kv_len that it
// had in the pool, or whatever the image holds there.
#pragma once
#include <algorithm>
#include <string>
#include <vector>

#include "common.h"

namespace vlo {

constexpr int kKvPageTokens = 64;

inline int kv_pages_for(long long tokens) { return static_cast<int>((tokens + kKvPageTokens - 1) / kKvPageTokens); }

class KvPool {
 public:
  int n_kv_heads = 0;
  int n_pages = 0;

  KvPool() = default;
  KvPool(const KvPool&) = delete;
  KvPool& operator=(const KvPool&) = delete;
  ~KvPool() {
    for (Gate& g : gates)
      if (g.ev) cudaEventDestroy(g.ev);
  }

  void init(int n_streams, int kv_heads, int pages) {
    n_kv_heads = kv_heads;
    n_pages = pages;
    for (int p = pages - 1; p >= 0; --p) free_list.push_back(p);  // page 0 first
    page_gate.assign(pages, -1);
    tables.assign(n_streams, {});
    lens.assign(n_streams, 0);
    opened.assign(n_streams, 0);
  }
  // rows between consecutive pages / kv heads in one layer's K or V matrix
  long long page_stride_rows() const { return static_cast<long long>(n_kv_heads) * kKvPageTokens; }
  static constexpr int head_stride_rows() { return kKvPageTokens; }
  long long rows_per_layer() const { return static_cast<long long>(n_pages) * page_stride_rows(); }
  // row of (cache position pos, kv head 0) of stream sid
  long long row(int sid, int pos) const {
    return tables[sid][pos / kKvPageTokens] * page_stride_rows() + pos % kKvPageTokens;
  }
  // pages on the free list, gated ones included
  int free_pages() const { return static_cast<int>(free_list.size()); }
  bool is_open(int sid) const { return opened[sid] != 0; }
  int len(int sid) const { return lens[sid]; }
  const std::vector<int>& table(int sid) const { return tables[sid]; }

  // open the first closed slot (an empty stream) as *sid
  int open(int* sid) {
    const auto it = std::find(opened.begin(), opened.end(), 0);
    if (it == opened.end()) return fail("no free stream slot (max_streams = " + std::to_string(opened.size()) + ")");
    *it = 1;
    *sid = static_cast<int>(it - opened.begin());
    return 0;
  }
  void close(int sid) {
    commit(sid, 0);
    opened[sid] = 0;
  }

  // Give streams sids[0..n) the pages to hold want[i] positions (a stream never loses pages here), all or none: a short
  // pool fails with nothing taken.  Stream st then waits for the swap-out copies that may still read a page taken, or
  // with `rewrite` any of the first ceil(want[i] / 64) pages (the call overwrites the stream from position 0).
  int grow(int n, const int* sids, const int* want, cudaStream_t st, bool rewrite = false) {
    int need = 0;
    for (int i = 0; i < n; ++i)
      need += std::max(0, kv_pages_for(want[i]) - static_cast<int>(tables[sids[i]].size()));
    if (need > free_pages())
      return fail("KV page pool exhausted: " + std::to_string(need) + " more pages of " + std::to_string(kKvPageTokens) +
                  " tokens needed, " + std::to_string(free_pages()) + " of " + std::to_string(n_pages) + " free");
    if (retire_gates()) return -1;
    std::vector<char> waited(gates.size(), 0);
    for (int i = 0; i < n; ++i) {
      std::vector<int>& t = tables[sids[i]];
      const size_t from = rewrite ? 0 : t.size(), pages = kv_pages_for(want[i]);
      grown.push_back(sids[i]);
      for (; t.size() < pages; free_list.pop_back()) t.push_back(free_list.back());
      for (size_t j = from; j < pages && live_gates > 0; ++j) {
        const int g = page_gate[t[j]];
        if (g < 0 || waited[g]) continue;
        VLO_CUDA(cudaStreamWaitEvent(st, gates[g].ev, 0));
        waited[g] = 1;
      }
    }
    return 0;
  }
  // Set stream sid's length once the work that writes its rows is enqueued; pages past ceil(len / 64) go back.
  void commit(int sid, int len) {
    lens[sid] = len;
    fit(sid);
  }
  // Return the pages grow() took and no commit() claimed: every table to ceil(len / 64), the free list as it was.
  void rollback() {
    for (auto s = grown.rbegin(); s != grown.rend(); ++s) fit(*s);
    grown.clear();
  }

  // Remove pages [first, first + n) from stream sid's table (full pages, the caller checks): they go back to the free
  // list, first on top; the later pages keep their rows and move n entries down, and the length drops by 64 n.
  void drop(int sid, int first, int n) {
    std::vector<int>& t = tables[sid];
    for (int j = first + n - 1; j >= first; --j) free_list.push_back(t[j]);
    t.erase(t.begin() + first, t.begin() + first + n);
    lens[sid] -= n * kKvPageTokens;
  }

  // Empty the non-empty stream sid once its swap-out copies are enqueued on st: its pages go back to the free list,
  // gated by an event recorded on st, and a grow() that takes one of them makes its stream wait on that event.
  int swap_out(int sid, cudaStream_t st) {
    if (retire_gates()) return -1;
    size_t g = 0;
    while (g < gates.size() && !gates[g].pages.empty()) ++g;
    if (g == gates.size()) gates.emplace_back();
    if (!gates[g].ev) VLO_CUDA(cudaEventCreateWithFlags(&gates[g].ev, cudaEventDisableTiming));
    VLO_CUDA(cudaEventRecord(gates[g].ev, st));
    gates[g].pages = tables[sid];
    for (int p : gates[g].pages) page_gate[p] = static_cast<int>(g);
    ++live_gates;
    commit(sid, 0);
    return 0;
  }

 private:
  struct Gate {
    cudaEvent_t ev = nullptr;
    std::vector<int> pages;  // empty: the gate is not live
  };
  std::vector<int> free_list;            // stack: back() is handed out next, released pages go back on top
  std::vector<std::vector<int>> tables;  // per stream slot: entry j = page of cache positions [64 j, 64 j + 64)
  std::vector<int> lens;                 // per stream slot: committed cache positions
  std::vector<char> opened;              // per stream slot
  std::vector<int> grown;                // streams grow() served since the last rollback(), in the order served
  std::vector<Gate> gates;
  std::vector<int> page_gate;            // gate page p waits for, or -1
  int live_gates = 0;

  // release the pages of stream sid past ceil(len / 64), last first
  void fit(int sid) {
    std::vector<int>& t = tables[sid];
    while (t.size() > static_cast<size_t>(kv_pages_for(lens[sid]))) {
      free_list.push_back(t.back());
      t.pop_back();
    }
  }
  // Release the gates whose swap-out copies have completed: their pages are ordinary free (or taken) pages again.
  int retire_gates() {
    for (size_t g = 0; g < gates.size() && live_gates > 0; ++g) {
      Gate& gate = gates[g];
      if (gate.pages.empty()) continue;
      const cudaError_t q = cudaEventQuery(gate.ev);
      if (q == cudaErrorNotReady) continue;
      VLO_CUDA(q);
      for (int p : gate.pages)
        if (page_gate[p] == static_cast<int>(g)) page_gate[p] = -1;
      gate.pages.clear();
      --live_gates;
    }
    return 0;
  }
};

// Scope of a call that grows streams: pages it took and did not commit go back when it returns, on every path.
struct KvGrowth {
  KvPool& pool;
  ~KvGrowth() { pool.rollback(); }
};

}  // namespace vlo
