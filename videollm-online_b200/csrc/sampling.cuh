// Response sampling on the device: sample_kernel draws one token id per bf16 logits row.
//
// Per row, in the order of HF's logits processors (GenerationMixin._get_logits_processor, transformers 5.5), in fp32 on
// the bf16 values:
//   1. repetition penalty over the row's id set: l = l < 0 ? l * p : l / p once for each distinct id of the set
//      (RepetitionPenaltyLogitsProcessor; ids outside [0, vocab) are ignored);
//   2. temperature: l = l / T (TemperatureLogitsWarper);
//   3. top-k: keep l >= the k-th largest l, so ties with the k-th value are kept (TopKLogitsWarper); k = 0 or k >= vocab
//      is off;
//   4. top-p: with p_i = softmax(l)_i over the top-k survivors, keep i iff the mass of the tokens with p_j > p_i
//      (strictly greater) is < top_p; top_p >= 1 is off.  A tie group that straddles the boundary is kept WHOLE: HF's
//      TopPLogitsWarper keeps the part of such a group its sort order puts first.  The maximum's tie group is always
//      kept (HF's min_tokens_to_keep = 1);
//   5. Gumbel-max draw: id = first-index argmax over the kept i of l_i + g_i, g_i = -log(-log(u_i)), with u_i from
//      counter-based Philox4x32-10 (layout in include/vlo_b200.h): a pure function of (seed, position, i).
//
// The id of a row is a function of its logits and parameters only: not of the rows beside it, of the SM that ran it or
// of the run.  So nothing is accumulated in floating point in scheduling order.  The top-k and top-p thresholds are found
// by a select over the order-preserving bit patterns of l (a histogram over 2048 linear value bins of the candidates,
// then four 8-bit radix digits inside the chosen bin) with integer counts and the probability mass in 2^-40 fixed point
// (u64 sums); min / max / argmax reductions are exact.  Every pass re-reads the row (256 KB at vocab 128 256, from L2)
// and recomputes l with the same operations, so each pass sees the same values; the digit levels read a compact copy of
// the chosen bin's candidates in shared memory instead when it fits.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

#include "ptx.cuh"

namespace vlo {

struct SampleRow {  // == vlo_sample_row
  unsigned long long seed;
  int position;
  float temperature;  // 0: the row is not sampled (id -1)
  int top_k;
  float top_p;
  float repetition_penalty;
  int penalty_offset, penalty_count;
  int reserved;
};
static_assert(sizeof(SampleRow) == 40, "SampleRow mirrors vlo_sample_row");

struct SampleInfo {  // per row, for the kernel-level entry: what the filters kept
  int kept;               // number of kept ids
  float topk_threshold;   // kept by top-k iff l >= this (-inf: off)
  float topp_threshold;   // kept by top-p iff l >= this (-inf: off)
  int reserved;
};

constexpr int kSampleThreads = 1024;
constexpr int kSampleBins = 2048;   // first-level value bins of the threshold select
constexpr float kSampleMassScale = 1099511627776.f;   // 2^40: fixed-point scale of exp(l - max)

// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

// g = -log(-log(u)), u = ((x >> 8) + 0.5) * 2^-24.  fp32 cannot hold u >= 0.5 exactly, so there -log(u) is computed as
// -log1p(-(1 - u)) from the exact 1 - u: the noise stays finite (at most about 17.3) and accurate to a few ulp.
__device__ __forceinline__ float gumbel_noise(uint32_t x) {
  const uint32_t k = x >> 8;
  const float e = k < (1u << 23) ? -logf((static_cast<float>(k) + 0.5f) * 0x1p-24f)
                                 : -log1pf(-(static_cast<float>((1u << 24) - 1u - k) + 0.5f) * 0x1p-24f);
  return -logf(e);
}

// order-preserving bit pattern of a float (larger float <-> larger key; +0 and -0 are made one value by the caller)
__device__ __forceinline__ uint32_t sample_key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float sample_key_value(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// l of element i (bf16 value x) after the penalty and the temperature; +0 for -0
struct SampleLogit {
  const uint32_t* bits;  // penalty set, one bit per id
  float penalty, temperature;
  __device__ __forceinline__ float operator()(int i, float x) const {
    float l = x;
    if (penalty != 1.f && ((bits[i >> 5] >> (i & 31)) & 1u)) l = l < 0.f ? l * penalty : l / penalty;
    l = l / temperature;
    return l == 0.f ? 0.f : l;
  }
};

// f(i, l) for every element of the row, 16-byte loads (vocab % 8 == 0)
template <typename F>
__device__ __forceinline__ void sample_sweep(const __nv_bfloat16* x, int vocab, const SampleLogit& lg, F&& f) {
  const int nvec = vocab / 8;
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    const uint4 raw = *reinterpret_cast<const uint4*>(x + static_cast<size_t>(v) * 8);
    const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 p = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[k]));
      f(v * 8 + 2 * k, lg(v * 8 + 2 * k, p.x));
      f(v * 8 + 2 * k + 1, lg(v * 8 + 2 * k + 1, p.y));
    }
  }
}

struct SampleShared {
  uint32_t cnt[kSampleBins];
  unsigned long long wt[kSampleBins];
  unsigned long long above;   // weight of the candidates above the current bucket range
  double target;              // weight the candidates above the threshold stay below
  int sel;                    // bucket chosen by sample_find
  int n_comp;                 // candidates of the chosen first-level bin copied to the compact list
  uint32_t red_u[32];
  float red_f[32];
  int red_i[32];
};

__device__ __forceinline__ uint32_t block_max_u32(uint32_t v, SampleShared& s) {
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s.red_u[threadIdx.x >> 5] = v;
  __syncthreads();
  v = s.red_u[0];
  for (int w = 1; w < static_cast<int>(blockDim.x >> 5); ++w) v = max(v, s.red_u[w]);
  return v;
}
__device__ __forceinline__ uint32_t block_min_u32(uint32_t v, SampleShared& s) {
  return ~block_max_u32(~v, s);
}

// Warp 0: among buckets [0, nb) (cnt / wt filled), the lowest non-empty bucket b whose candidates above it
// (s.above + weight of buckets > b) weigh less than s.target; s.sel = b, s.above += weight of buckets > b.
// The condition holds for every b from some b0 up, so b is the bucket of the threshold of a descending walk.
// target_frac >= 0 (first level only): s.target = target_frac * the total weight of the buckets.
__device__ __forceinline__ void sample_find(SampleShared& s, int nb, double target_frac = -1.0) {
  __syncthreads();
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x, per = nb / 32, base = lane * per;
    unsigned long long mine = 0;
    for (int j = 0; j < per; ++j) mine += s.wt[base + j];
    unsigned long long suf = mine;   // weight of the buckets of lanes >= lane
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long t = __shfl_down_sync(0xffffffffu, suf, o);
      if (lane + o < 32) suf += t;
    }
    const double target =
        target_frac >= 0.0 ? target_frac * static_cast<double>(__shfl_sync(0xffffffffu, suf, 0)) : s.target;
    unsigned long long acc = s.above + (suf - mine), best_acc = 0;
    int best = 0x7fffffff;
    for (int j = per - 1; j >= 0; --j) {
      const int b = base + j;
      if (s.cnt[b] > 0 && static_cast<double>(acc) < target) {
        best = b;
        best_acc = acc;
      }
      acc += s.wt[b];
    }
    int b = best;
    for (int o = 16; o > 0; o >>= 1) b = min(b, __shfl_xor_sync(0xffffffffu, b, o));
    const unsigned long long a = __shfl_sync(0xffffffffu, best_acc, (b == 0x7fffffff ? 0 : b / per));
    if (lane == 0) {
      s.sel = b;
      s.above = a;
      s.target = target;
    }
  }
  __syncthreads();
}

// The threshold key among the candidates (key >= floor_key, keys within [lo_key, hi_key]): walking them in descending
// order, with weight 1 each (kMass false) or the fixed-point mass of exp(l - m) (kMass true), the smallest key whose
// strictly greater candidates weigh less than the target: k in count mode (the k-th largest key), top_p times their
// total mass in mass mode.
template <bool kMass>
__device__ uint32_t sample_select(const __nv_bfloat16* x, int vocab, const SampleLogit& lg, uint32_t floor_key,
                                  uint32_t lo_key, uint32_t hi_key, float m, double target, SampleShared& s) {
  const float lo = sample_key_value(lo_key), hi = sample_key_value(hi_key);
  const bool flat = !(hi - lo >= 1e-30f);
  const float scale = flat ? 0.f : static_cast<float>(kSampleBins) / (hi - lo);
  auto bin = [&](float l) { return flat ? 0 : min(kSampleBins - 1, static_cast<int>((l - lo) * scale)); };
  auto weight = [&](float l) -> unsigned long long {
    return kMass ? __float2ull_rz(expf(l - m) * kSampleMassScale) : 1ull;
  };
  // level 1: value bins
  for (int b = threadIdx.x; b < kSampleBins; b += blockDim.x) {
    s.cnt[b] = 0;
    s.wt[b] = 0;
  }
  if (threadIdx.x == 0) {
    s.above = 0;
    s.target = target;
    s.n_comp = 0;
  }
  __syncthreads();
  sample_sweep(x, vocab, lg, [&](int, float l) {
    if (sample_key(l) < floor_key) return;
    const int b = bin(l);
    atomicAdd(&s.cnt[b], 1u);
    atomicAdd(&s.wt[b], weight(l));
  });
  sample_find(s, kSampleBins, kMass ? target : -1.0);
  const int sel_bin = s.sel;
  // The chosen bin's candidates (key, weight) go to a compact list in the unused tail of cnt / wt when they fit, so
  // that the digit levels read shared memory instead of the row; the list's order does not matter to the counts.
  uint32_t* ck = s.cnt + 256;
  unsigned long long* cw = s.wt + 256;
  const bool compact = s.cnt[sel_bin] <= static_cast<uint32_t>(kSampleBins - 256);
  __syncthreads();
  if (compact)
    sample_sweep(x, vocab, lg, [&](int, float l) {
      const uint32_t k = sample_key(l);
      if (k < floor_key || bin(l) != sel_bin) return;
      const int j = atomicAdd(&s.n_comp, 1);
      ck[j] = k;
      cw[j] = weight(l);
    });
  // levels 2-5: 8-bit digits of the key inside that bin
  uint32_t prefix = 0, mask = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int b = threadIdx.x; b < 256; b += blockDim.x) {
      s.cnt[b] = 0;
      s.wt[b] = 0;
    }
    __syncthreads();
    if (compact) {
      for (int j = threadIdx.x; j < s.n_comp; j += blockDim.x) {
        const uint32_t k = ck[j];
        if ((k & mask) != prefix) continue;
        atomicAdd(&s.cnt[(k >> shift) & 255], 1u);
        atomicAdd(&s.wt[(k >> shift) & 255], cw[j]);
      }
    } else {
      sample_sweep(x, vocab, lg, [&](int, float l) {
        const uint32_t k = sample_key(l);
        if (k < floor_key || (k & mask) != prefix || bin(l) != sel_bin) return;
        const int d = (k >> shift) & 255;
        atomicAdd(&s.cnt[d], 1u);
        atomicAdd(&s.wt[d], weight(l));
      });
    }
    sample_find(s, 256);
    prefix |= static_cast<uint32_t>(s.sel) << shift;
    mask |= 255u << shift;
  }
  return prefix;
}

// One block per row.  rows / penalty_ids: device copies of the call's parameters; info may be null.
// Dynamic shared memory: the penalty bit set, ceil(vocab / 32) words.
__global__ void __launch_bounds__(kSampleThreads) sample_kernel(const __nv_bfloat16* logits, int vocab,
                                                                const SampleRow* rows, const int* penalty_ids,
                                                                int* out_ids, SampleInfo* info) {
  extern __shared__ uint32_t s_bits[];
  __shared__ SampleShared s;
  pdl_trigger();
  // the parameters come from a memcpy enqueued before this kernel: readable before the grid dependency resolves
  const SampleRow r = rows[blockIdx.x];
  if (r.temperature == 0.f) {
    if (threadIdx.x == 0) {
      pdl_wait();
      out_ids[blockIdx.x] = -1;
      if (info) info[blockIdx.x] = SampleInfo{0, -INFINITY, -INFINITY, 0};
    }
    return;
  }
  const int n_words = (vocab + 31) / 32;
  for (int w = threadIdx.x; w < n_words; w += blockDim.x) s_bits[w] = 0;
  __syncthreads();
  if (r.repetition_penalty != 1.f)
    for (int j = threadIdx.x; j < r.penalty_count; j += blockDim.x) {
      const int id = penalty_ids[r.penalty_offset + j];
      if (id >= 0 && id < vocab) atomicOr(&s_bits[id >> 5], 1u << (id & 31));
    }
  __syncthreads();
  pdl_wait();
  const __nv_bfloat16* x = logits + static_cast<size_t>(blockIdx.x) * vocab;
  const SampleLogit lg{s_bits, r.repetition_penalty, r.temperature};
  const bool use_k = r.top_k > 0 && r.top_k < vocab, use_p = r.top_p < 1.f;

  uint32_t thr = 0, thr_k = 0, thr_p = 0;   // kept iff key >= thr (0: everything)
  if (use_k || use_p) {
    uint32_t kmax = 0, kmin = 0xffffffffu;
    sample_sweep(x, vocab, lg, [&](int, float l) {
      const uint32_t k = sample_key(l);
      kmax = max(kmax, k);
      kmin = min(kmin, k);
    });
    kmax = block_max_u32(kmax, s);
    kmin = block_min_u32(kmin, s);
    const float m = sample_key_value(kmax);
    if (use_k) thr = thr_k = sample_select<false>(x, vocab, lg, 0u, kmin, kmax, m, static_cast<double>(r.top_k), s);
    if (use_p) {
      // the top-p threshold among the top-k survivors, against top_p times their total mass
      thr = thr_p = sample_select<true>(x, vocab, lg, thr, max(thr, kmin), kmax, m, static_cast<double>(r.top_p), s);
    }
  }

  // Gumbel-max draw over the kept ids; noise word i % 4 of Philox(counter (i / 4, position, 0, 0), key seed)
  const uint32_t k0 = static_cast<uint32_t>(r.seed), k1 = static_cast<uint32_t>(r.seed >> 32);
  float best = -INFINITY;
  int best_i = 0x7fffffff, kept = 0;
  const int nvec = vocab / 8;
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    const uint4 raw = *reinterpret_cast<const uint4*>(x + static_cast<size_t>(v) * 8);
    const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
    float l[8];
    bool any[2] = {false, false};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 p = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[k]));
      l[2 * k] = lg(v * 8 + 2 * k, p.x);
      l[2 * k + 1] = lg(v * 8 + 2 * k + 1, p.y);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) any[j >> 2] |= sample_key(l[j]) >= thr;
#pragma unroll
    for (int g = 0; g < 2; ++g) {
      if (!any[g]) continue;
      const uint4 n = philox4x32_10(make_uint4(static_cast<uint32_t>(2 * v + g), static_cast<uint32_t>(r.position), 0u, 0u),
                                    k0, k1);
      const uint32_t word[4] = {n.x, n.y, n.z, n.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float lj = l[4 * g + j];
        if (sample_key(lj) < thr) continue;
        ++kept;
        const float sc = lj + gumbel_noise(word[j]);
        if (sc > best) {   // indices rise within a thread: the first index wins a tie
          best = sc;
          best_i = v * 8 + 4 * g + j;
        }
      }
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
    kept += __shfl_xor_sync(0xffffffffu, kept, o);
    if (ob > best || (ob == best && oi < best_i)) {
      best = ob;
      best_i = oi;
    }
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) {
    s.red_f[threadIdx.x >> 5] = best;
    s.red_i[threadIdx.x >> 5] = best_i;
    s.red_u[threadIdx.x >> 5] = static_cast<uint32_t>(kept);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    best = s.red_f[0];
    best_i = s.red_i[0];
    uint32_t n_kept = s.red_u[0];
    for (int w = 1; w < static_cast<int>(blockDim.x >> 5); ++w) {
      if (s.red_f[w] > best || (s.red_f[w] == best && s.red_i[w] < best_i)) {
        best = s.red_f[w];
        best_i = s.red_i[w];
      }
      n_kept += s.red_u[w];
    }
    out_ids[blockIdx.x] = best_i;
    if (info)
      info[blockIdx.x] = SampleInfo{static_cast<int>(n_kept), use_k ? sample_key_value(thr_k) : -INFINITY,
                                    use_p ? sample_key_value(thr_p) : -INFINITY, 0};
  }
}

}  // namespace vlo
