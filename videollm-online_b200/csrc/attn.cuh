// KV-append attention for the decoder (SURVEY K15): causal-with-offset GQA attention of a few new
// query tokens (q = 1 AR token, 11 frame-step tokens, a short prompt) over ALL cached keys.
// Replaces HF:models/llama/modeling_llama.py:272-285 (SDPA / flash-attn-2) for the KV-append case.
//
// Memory-bound by design: per kv head the K and V rows ([key][128] bf16, 256 B each) are streamed
// from HBM exactly once by TMA into 128B-swizzled shared memory; the G = n_heads/n_kv_heads query
// heads x q tokens that share a kv head form one <=64-row tile so every K/V byte is reused
// G*q times from shared memory.  The key range is split across CTAs (split-KV) and inside a CTA
// across two warp groups; partial (max, sum, O) triples are merged by attn_merge_kernel.
//   v1 math: mma.sync m16n8k16 bf16 (fp32 accumulate), online softmax in registers.
#pragma once
#include <cuda.h>
#include "ptx.cuh"
#include "mma.cuh"

namespace vlo {

constexpr int kAttnHD = 128;       // head_dim (Llama-3)
constexpr int kAttnBlk = 64;       // keys per pipeline stage
constexpr int kAttnStages = 3;     // per warp group
constexpr int kAttnGroups = 2;     // warp groups per CTA, alternate key blocks
constexpr int kAttnThreads = 32 * (1 + 4 * kAttnGroups);  // 1 producer warp + 8 MMA warps
constexpr int kAttnSubTile = kAttnBlk * 128;               // 64 keys x 64 dims x 2 B = 8 KB
constexpr int kAttnStageBytes = 4 * kAttnSubTile;          // K(2 halves) + V(2 halves) = 32 KB
constexpr int kAttnSmemBase = kAttnGroups * kAttnStages * kAttnStageBytes + 1024 + 256;  // ring + alignment + barriers
constexpr int kAttnSmemOptIn = 232448;  // 227 KB: the per-block dynamic shared memory limit of sm_90
// All of a split's page-table entries (4 B each) are staged in shared memory behind the barriers before the grid
// dependency resolves, so the TMA producer issues every key block without a global load.  A launch sizes that area for
// the plan's longest split (attn_smem_bytes); the opt-in limit leaves room for kAttnPtMax entries (552 960 keys).
constexpr int kAttnPtMax = (kAttnSmemOptIn - kAttnSmemBase) / 4;
inline int attn_smem_bytes(int max_blocks_per_split) { return kAttnSmemBase + 4 * max_blocks_per_split; }

// Key block b (64 keys) of kv head h of an item lives at row page_table[pt0 + b] * page_stride_rows + h * head_stride_rows
// of the K / V maps (rows in units of head_dim elements).  The engine's page pool has page_stride_rows = n_kv_heads * 64
// and head_stride_rows = 64; a contiguous [n_kv_heads][stride][128] cache is an identity table with page_stride_rows = 64
// and head_stride_rows = stride.
struct AttnItem {
  int q_tok0;          // first token of this chunk in the packed q / out arrays
  int q_count;         // tokens in the chunk; q_count * G <= 64
  int q_pos0;          // absolute position of the chunk's first token (= #keys strictly before it)
  int pt0;             // page-table entry of the sequence's key block 0
  int n_splits;        // splits that own at least one key block
  int blocks_per_split;
  int ws_slot0;        // first workspace row-slot of this item
};

struct AttnParams {
  const __nv_bfloat16* q;  // [n_tok, n_heads, 128], RoPE applied
  float* ws_o;             // [slots, 128] un-normalised partial outputs
  float* ws_ml;            // [slots, 2]   (row max in raw-score units, row sum)
  const AttnItem* items;
  const int* page_table;   // page of each 64-key block, per sequence from AttnItem::pt0
  int page_stride_rows, head_stride_rows;
  int n_heads, n_kv_heads;
  float scale_log2;        // head_dim^-0.5 * log2(e)
};

// One CTA of the KV-append attention: item `it`, key split `split`, kv head `kvh`.
// kCluster = false: attn_kvappend_kernel, the CTA loads its own key blocks.
// kCluster = true: attn_kvappend_cluster_kernel, one CTA per item of a cluster of items of ONE stream with the same
//   blocks_per_split, all on the same (split, kv head).  The cluster loads nblk_load >= nblk key blocks (the longest
//   member's); block b is loaded by CTA b % cs with a TMA multicast into the same ring stage of every CTA, so the cache
//   crosses HBM -> L2 -> SM once per cluster.  A stage is refilled only when every CTA has released it: each producer,
//   once its own MMA warps released a stage, arrives on the cluster-release barrier of every CTA, and the loading CTA
//   waits on its own.  The MMA warps run the same code on the blocks of their own item and only take part in the ring
//   protocol on the others; a CTA that is not `active` (its item has no block in this split, or a padding rank) writes
//   nothing.
// kPacked = true: attn_kvappend_packed_kernel, `it` spans a run of it.q_count consecutive one-token segments whose items
//   are p.items[item0 ..] and share n_splits and blocks_per_split.  Row r is token r / G of the run, as in a multi-token
//   item, and it produces the bits of its own segment's item: it skips the key blocks past its own position (its solo
//   item has none of them; a fully masked block is not a no-op, the rescale FMA need not be exactly 1), and it writes
//   its partial to that item's slots.
template <bool kCluster, bool kPacked = false>
__device__ __forceinline__ void attn_kvappend_cta(const CUtensorMap& tm_k, const CUtensorMap& tm_v, const AttnParams& p,
                                                  const AttnItem& it, int split, int kvh, int nblk_load, bool active,
                                                  uint32_t rank, uint32_t cs, int item0 = 0) {
  const int G = p.n_heads / p.n_kv_heads;
  const int rows = it.q_count * G;
  const int mt_active = (rows + 15) >> 4;  // MMA warps per group that own real rows
  const int kv_end = it.q_pos0 + it.q_count;
  const int nblk_total = (kv_end + kAttnBlk - 1) / kAttnBlk;
  const int blk0 = split * it.blocks_per_split;
  const int blk1 = min(blk0 + it.blocks_per_split, nblk_total);
  const int nblk = kCluster ? (active ? blk1 - blk0 : 0) : blk1 - blk0;
  const int nblk_ld = kCluster ? nblk_load : nblk;  // key blocks that go through this CTA's ring

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kAttnGroups * kAttnStages * kAttnStageBytes);
  uint64_t* empty_bar = full_bar + kAttnGroups * kAttnStages;
  uint64_t* cl_empty_bar = empty_bar + kAttnGroups * kAttnStages;  // cluster release (kCluster only)
  int* s_pt = reinterpret_cast<int*>(smem + kAttnGroups * kAttnStages * kAttnStageBytes + 256);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j = threadIdx.x; j < nblk_ld; j += kAttnThreads) s_pt[j] = p.page_table[it.pt0 + blk0 + j];
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    for (int i = 0; i < kAttnGroups * kAttnStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], mt_active);
      if (kCluster) mbar_init(&cl_empty_bar[i], cs);
    }
    fence_mbar_init();
  }
  pdl_wait();   // the freshly appended K/V rows and Q come from predecessors
  __syncthreads();
  if (kCluster) cluster_sync();  // every CTA's barriers are initialised before any multicast or remote arrive

  const int head_row = kvh * p.head_stride_rows;

  // MMA-warp state (also declared for the producer warp; unused there)
  float o_acc[16][4];
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 16; ++i) o_acc[i][0] = o_acc[i][1] = o_acc[i][2] = o_acc[i][3] = 0.f;

  const int cw = warp - 1;           // 0..7 for MMA warps
  const int grp = cw >> 2;           // warp group
  const int mt = cw & 3;             // m-tile (16 rows) owned by this warp
  const int g8 = lane >> 2, q4 = lane & 3;

  if (warp == 0) {
    if (lane == 0) {
      // ---------------------------------------------------------- TMA producer
      for (int b = 0; b < nblk_ld; ++b) {
        const int g = b & 1;
        const int i = b >> 1;
        const int s = i % kAttnStages;
        const uint32_t ph = (i / kAttnStages) & 1;
        uint64_t* fb = &full_bar[g * kAttnStages + s];
        mbar_wait(&empty_bar[g * kAttnStages + s], ph ^ 1);
        if (kCluster && i >= kAttnStages)  // this CTA released the stage's previous block: tell every CTA of the cluster
          for (uint32_t r = 0; r < cs; ++r) mbar_arrive_cluster(&cl_empty_bar[g * kAttnStages + s], r);
        mbar_arrive_expect_tx(fb, kAttnStageBytes);  // cluster: peers' copies may land before this, the phase waits for it
        uint8_t* st = smem + (g * kAttnStages + s) * kAttnStageBytes;
        const int row = s_pt[b] * p.page_stride_rows + head_row;
        if (kCluster) {
          if (static_cast<uint32_t>(b) % cs == rank) {
            mbar_wait(&cl_empty_bar[g * kAttnStages + s], ph ^ 1);  // every CTA released the stage
            const uint16_t mask = static_cast<uint16_t>((1u << cs) - 1);
            tma_load_2d_multicast(st, &tm_k, fb, 0, row, mask, kEvictFirst);
            tma_load_2d_multicast(st + kAttnSubTile, &tm_k, fb, 64, row, mask, kEvictFirst);
            tma_load_2d_multicast(st + 2 * kAttnSubTile, &tm_v, fb, 0, row, mask, kEvictFirst);
            tma_load_2d_multicast(st + 3 * kAttnSubTile, &tm_v, fb, 64, row, mask, kEvictFirst);
          }
        } else {
          tma_load_2d(st, &tm_k, fb, 0, row, kEvictFirst);
          tma_load_2d(st + kAttnSubTile, &tm_k, fb, 64, row, kEvictFirst);
          tma_load_2d(st + 2 * kAttnSubTile, &tm_v, fb, 0, row, kEvictFirst);
          tma_load_2d(st + 3 * kAttnSubTile, &tm_v, fb, 64, row, kEvictFirst);
        }
      }
    }
  } else if (mt < mt_active) {
    // ------------------------------------------------------------ MMA warps
    // Q fragments for this warp's 16 rows: row r = t * G + g  (t token, g head in the kv group).
    uint32_t qf[8][4];
    {
      const int r0 = mt * 16 + g8, r1 = r0 + 8;
      const __nv_bfloat16* q0 = nullptr;
      const __nv_bfloat16* q1 = nullptr;
      if (r0 < rows)
        q0 = p.q + (static_cast<size_t>(it.q_tok0 + r0 / G) * p.n_heads + kvh * G + (r0 % G)) * kAttnHD;
      if (r1 < rows)
        q1 = p.q + (static_cast<size_t>(it.q_tok0 + r1 / G) * p.n_heads + kvh * G + (r1 % G)) * kAttnHD;
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        const int c = ks * 16 + q4 * 2;
        qf[ks][0] = q0 ? *reinterpret_cast<const uint32_t*>(q0 + c) : 0u;
        qf[ks][1] = q1 ? *reinterpret_cast<const uint32_t*>(q1 + c) : 0u;
        qf[ks][2] = q0 ? *reinterpret_cast<const uint32_t*>(q0 + c + 8) : 0u;
        qf[ks][3] = q1 ? *reinterpret_cast<const uint32_t*>(q1 + c + 8) : 0u;
      }
    }
    const int r0 = mt * 16 + g8, r1 = r0 + 8;
    // last visible key per row (causal with offset); padding rows see nothing.
    const int lim0 = r0 < rows ? it.q_pos0 + r0 / G : -1;
    const int lim1 = r1 < rows ? it.q_pos0 + r1 / G : -1;
    const float c = p.scale_log2;

    for (int b = grp; b < nblk_ld; b += kAttnGroups) {
      const int i = b >> 1;
      const int s = i % kAttnStages;
      const uint32_t ph = (i / kAttnStages) & 1;
      mbar_wait(&full_bar[grp * kAttnStages + s], ph);
      if (kCluster && b >= nblk) {  // a block of a longer member of the cluster: release it untouched
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[grp * kAttnStages + s]);
        continue;
      }
      const uint32_t st = smem_u32(smem + (grp * kAttnStages + s) * kAttnStageBytes);
      const int key0 = (blk0 + b) * kAttnBlk;

      // S = Q K^T  (16 x 64)
      float sc[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
        const int krow = nt * 8 + (lane & 7);
#pragma unroll
        for (int kp = 0; kp < 4; ++kp) {  // pairs of k-steps (32 dims)
          const int cg = kp * 4 + (lane >> 3);  // 16-byte chunk 0..15 along head_dim
          const uint32_t addr = st + (cg >> 3) * kAttnSubTile + krow * 128 + (((cg & 7) ^ (krow & 7)) << 4);
          uint32_t b0, b1, b2, b3;
          ldsm_x4(addr, b0, b1, b2, b3);
          mma_bf16_16816(sc[nt], qf[2 * kp], b0, b1);
          mma_bf16_16816(sc[nt], qf[2 * kp + 1], b2, b3);
        }
      }
      // causal / length mask (only blocks that reach past the first query's limit)
      if (key0 + kAttnBlk - 1 > it.q_pos0) {
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          const int k = key0 + nt * 8 + q4 * 2;
          if (k > lim0) sc[nt][0] = -INFINITY;
          if (k + 1 > lim0) sc[nt][1] = -INFINITY;
          if (k > lim1) sc[nt][2] = -INFINITY;
          if (k + 1 > lim1) sc[nt][3] = -INFINITY;
        }
      } else if (lim0 < 0 || lim1 < 0) {
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          if (lim0 < 0) sc[nt][0] = sc[nt][1] = -INFINITY;
          if (lim1 < 0) sc[nt][2] = sc[nt][3] = -INFINITY;
        }
      }
      // online softmax
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        mx0 = fmaxf(mx0, fmaxf(sc[nt][0], sc[nt][1]));
        mx1 = fmaxf(mx1, fmaxf(sc[nt][2], sc[nt][3]));
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      const float mn0 = fmaxf(m_run[0], mx0), mn1 = fmaxf(m_run[1], mx1);
      const float me0 = (mn0 == -INFINITY) ? 0.f : mn0 * c;
      const float me1 = (mn1 == -INFINITY) ? 0.f : mn1 * c;
      // kPacked: a row past its own last block keeps (m, l, O): its scores are all -inf, so m stays, its P row is 0,
      // and the rescale is selected to exactly 1 instead of computed
      const bool in0 = !kPacked || key0 <= lim0, in1 = !kPacked || key0 <= lim1;
      const float al0 = in0 ? exp2f(m_run[0] * c - me0) : 1.f, al1 = in1 ? exp2f(m_run[1] * c - me1) : 1.f;
      m_run[0] = mn0;
      m_run[1] = mn1;
      float ps0 = 0.f, ps1 = 0.f;
      uint32_t pf[4][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const float p0 = exp2f(sc[nt][0] * c - me0), p1 = exp2f(sc[nt][1] * c - me0);
        const float p2 = exp2f(sc[nt][2] * c - me1), p3 = exp2f(sc[nt][3] * c - me1);
        ps0 += p0 + p1;
        ps1 += p2 + p3;
        pf[nt >> 1][(nt & 1) * 2 + 0] = pack_bf16(p0, p1);
        pf[nt >> 1][(nt & 1) * 2 + 1] = pack_bf16(p2, p3);
      }
      // explicit FMAs (the fusion attn_kvappend_kernel gets): see the warp-group merge below
      l_run[0] = __fmaf_rn(l_run[0], al0, ps0);
      l_run[1] = __fmaf_rn(l_run[1], al1, ps1);
#pragma unroll
      for (int nd = 0; nd < 16; ++nd) {
        o_acc[nd][0] *= al0;
        o_acc[nd][1] *= al0;
        o_acc[nd][2] *= al1;
        o_acc[nd][3] *= al1;
      }
      // The block that holds kv_end loads rows past it: stale rows of a reused page or this stream's rows left past a
      // truncate, evict or compact.  Their P is exactly 0, but 0 * Inf and 0 * NaN are NaN, so the group's warps zero
      // those V rows in the stage before the P V product reads it.  A finite row's 0 * v adds nothing, so the bits stay
      // those of the unmasked product; every other block skips this branch (the test is block-uniform).
      if (key0 + kAttnBlk > kv_end) {
        uint8_t* vst = smem + (grp * kAttnStages + s) * kAttnStageBytes + 2 * kAttnSubTile;
        const int first = kv_end - key0;  // rows first .. 63 of both 64-dim halves: 16 chunks of 16 B per row
        for (int c = mt * 32 + lane; c < (kAttnBlk - first) * 16; c += mt_active * 32) {
          const int row = first + (c >> 4), ch = c & 15;
          *reinterpret_cast<uint4*>(vst + (ch >> 3) * kAttnSubTile + row * 128 + (ch & 7) * 16) = make_uint4(0, 0, 0, 0);
        }
        fence_proxy_async();                       // the stage's next TMA fill is ordered after these stores
        if (grp == 0)                              // every warp of the group sees the whole cleared tail
          named_bar_sync<1>(mt_active * 32);
        else
          named_bar_sync<2>(mt_active * 32);
      }
      // O += P V   (16 x 128), V tile rows = keys, transposed ldmatrix
      const uint32_t sv = st + 2 * kAttnSubTile;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const int vrow = kk * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
#pragma unroll
        for (int np = 0; np < 8; ++np) {  // pairs of 8-wide d tiles
          const int cg = np * 2 + (lane >> 4);
          const uint32_t addr = sv + (cg >> 3) * kAttnSubTile + vrow * 128 + (((cg & 7) ^ (vrow & 7)) << 4);
          uint32_t b0, b1, b2, b3;
          ldsm_x4_t(addr, b0, b1, b2, b3);
          mma_bf16_16816(o_acc[2 * np], pf[kk], b0, b1);
          mma_bf16_16816(o_acc[2 * np + 1], pf[kk], b2, b3);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[grp * kAttnStages + s]);
    }
    l_run[0] += __shfl_xor_sync(0xffffffffu, l_run[0], 1);
    l_run[0] += __shfl_xor_sync(0xffffffffu, l_run[0], 2);
    l_run[1] += __shfl_xor_sync(0xffffffffu, l_run[1], 1);
    l_run[1] += __shfl_xor_sync(0xffffffffu, l_run[1], 2);
  }

  // ---- merge the two warp groups through shared memory (pipeline buffers are idle now)
  __syncthreads();
  if (kCluster && !active) return;  // the caller's cluster_sync follows
  float* xo = reinterpret_cast<float*>(smem);            // [4 warps][16 rows][128]
  float* xml = xo + 4 * 16 * kAttnHD;                     // [4 warps][16 rows][2]
  if (warp > 0 && mt < mt_active && grp == 1) {
    float* wo = xo + mt * 16 * kAttnHD;
#pragma unroll
    for (int nd = 0; nd < 16; ++nd) {
      *reinterpret_cast<float2*>(wo + g8 * kAttnHD + nd * 8 + q4 * 2) = make_float2(o_acc[nd][0], o_acc[nd][1]);
      *reinterpret_cast<float2*>(wo + (g8 + 8) * kAttnHD + nd * 8 + q4 * 2) = make_float2(o_acc[nd][2], o_acc[nd][3]);
    }
    if (q4 == 0) {
      xml[(mt * 16 + g8) * 2 + 0] = m_run[0];
      xml[(mt * 16 + g8) * 2 + 1] = l_run[0];
      xml[(mt * 16 + g8 + 8) * 2 + 0] = m_run[1];
      xml[(mt * 16 + g8 + 8) * 2 + 1] = l_run[1];
    }
  }
  __syncthreads();
  if (warp > 0 && mt < mt_active && grp == 0) {
    const float c = p.scale_log2;
    const float* wo = xo + mt * 16 * kAttnHD;
    const float om0 = xml[(mt * 16 + g8) * 2], ol0 = xml[(mt * 16 + g8) * 2 + 1];
    const float om1 = xml[(mt * 16 + g8 + 8) * 2], ol1 = xml[(mt * 16 + g8 + 8) * 2 + 1];
    const float mn0 = fmaxf(m_run[0], om0), mn1 = fmaxf(m_run[1], om1);
    const float me0 = (mn0 == -INFINITY) ? 0.f : mn0 * c, me1 = (mn1 == -INFINITY) ? 0.f : mn1 * c;
    const float a0 = exp2f(m_run[0] * c - me0), b0 = exp2f(om0 * c - me0);
    const float a1 = exp2f(m_run[1] * c - me1), b1 = exp2f(om1 * c - me1);
    // Rounding spelled out: attn_kvappend_kernel computes the first eight rows of an m-tile (r0) without an FMA and the
    // second eight (r1) with one, as the compiler fused them there.  A packed row must take the form its own one-token
    // item uses: with G <= 8 that item's rows are all r0 rows.
    const float l0 = __fadd_rn(__fmul_rn(l_run[0], a0), __fmul_rn(ol0, b0));
    const float l1 = kPacked && G <= 8 ? __fadd_rn(__fmul_rn(l_run[1], a1), __fmul_rn(ol1, b1))
                                       : __fmaf_rn(l_run[1], a1, __fmul_rn(ol1, b1));
    const int r0 = mt * 16 + g8, r1 = r0 + 8;
    const size_t slot_base = static_cast<size_t>(it.ws_slot0) +
                             (static_cast<size_t>(kvh) * it.n_splits + split) * rows;
    // kPacked: row r is row r % G of the one-token item item0 + r / G (G rows per item, the run's n_splits)
    auto packed_slot = [&](int r) {
      const int G = p.n_heads / p.n_kv_heads;
      return static_cast<size_t>(p.items[item0 + r / G].ws_slot0) +
             (static_cast<size_t>(kvh) * it.n_splits + split) * G + r % G;
    };
    size_t pslot0 = 0, pslot1 = 0;
    if constexpr (kPacked) {
      if (r0 < rows) pslot0 = packed_slot(r0);
      if (r1 < rows) pslot1 = packed_slot(r1);
    }
#pragma unroll
    for (int nd = 0; nd < 16; ++nd) {
      const float2 x0 = *reinterpret_cast<const float2*>(wo + g8 * kAttnHD + nd * 8 + q4 * 2);
      const float2 x1 = *reinterpret_cast<const float2*>(wo + (g8 + 8) * kAttnHD + nd * 8 + q4 * 2);
      if (r0 < rows)
        *reinterpret_cast<float2*>(p.ws_o + (kPacked ? pslot0 : slot_base + r0) * kAttnHD + nd * 8 + q4 * 2) =
            make_float2(o_acc[nd][0] * a0 + x0.x * b0, o_acc[nd][1] * a0 + x0.y * b0);
      if (r1 < rows)
        *reinterpret_cast<float2*>(p.ws_o + (kPacked ? pslot1 : slot_base + r1) * kAttnHD + nd * 8 + q4 * 2) =
            make_float2(o_acc[nd][2] * a1 + x1.x * b1, o_acc[nd][3] * a1 + x1.y * b1);
    }
    if (q4 == 0) {
      if (r0 < rows) {
        p.ws_ml[(kPacked ? pslot0 : slot_base + r0) * 2] = mn0;
        p.ws_ml[(kPacked ? pslot0 : slot_base + r0) * 2 + 1] = l0;
      }
      if (r1 < rows) {
        p.ws_ml[(kPacked ? pslot1 : slot_base + r1) * 2] = mn1;
        p.ws_ml[(kPacked ? pslot1 : slot_base + r1) * 2 + 1] = l1;
      }
    }
  }
}


// grid = (max_splits, n_kv_heads, n_items); block = kAttnThreads.
__global__ void __launch_bounds__(kAttnThreads, 1)
attn_kvappend_kernel(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v,
                     const AttnParams p) {
  pdl_trigger();
  // The item table and the page tables were uploaded by the memcpy at the start of the step: they (and this split's
  // page entries, below) are read before the grid dependency resolves.
  const AttnItem it = p.items[blockIdx.z];
  const int split = blockIdx.x;
  if (split >= it.n_splits) return;
  attn_kvappend_cta<false>(tm_k, tm_v, p, it, split, blockIdx.y, 0, true, 0, 1);
}

constexpr int kAttnClusterMax = 8;  // portable cluster size
// members of one cluster: item indices, -1 for the padding ranks of a cluster smaller than the launch's cluster size
struct AttnCluster {
  int item[kAttnClusterMax];
};

// grid = (cs * n_clusters, max_splits, n_kv_heads), cluster = (cs, 1, 1); block = kAttnThreads.
__global__ void __launch_bounds__(kAttnThreads, 1)
attn_kvappend_cluster_kernel(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v,
                             const AttnParams p, const AttnCluster* clusters) {
  pdl_trigger();
  const uint32_t cs = cluster_nctarank();
  const uint32_t rank = cluster_ctarank();
  const AttnCluster& cl = clusters[blockIdx.x / cs];
  const int split = blockIdx.y;
  // blocks the cluster loads in this split: the longest member's (all members share blocks_per_split)
  int nblk_load = 0;
  for (uint32_t r = 0; r < cs; ++r) {
    const int m = cl.item[r];
    if (m < 0) continue;
    const AttnItem& im = p.items[m];
    if (split >= im.n_splits) continue;
    const int nb = (im.q_pos0 + im.q_count + kAttnBlk - 1) / kAttnBlk;
    nblk_load = max(nblk_load, min(im.blocks_per_split, nb - split * im.blocks_per_split));
  }
  if (nblk_load == 0) return;  // no member has this split: the whole cluster leaves together
  const int own = cl.item[rank];
  const AttnItem it = p.items[own >= 0 ? own : cl.item[0]];
  attn_kvappend_cta<true>(tm_k, tm_v, p, it, split, blockIdx.z, nblk_load, own >= 0 && split < it.n_splits, rank, cs);
  cluster_sync();  // no CTA leaves while another may still arrive on its barriers
}

// A run of `count` (2 .. 64 / G) consecutive one-token segments of one sequence: items item0 .. item0 + count - 1, in
// order, all with the same n_splits and blocks_per_split.
struct AttnPack {
  int item0, count;
};

// grid = (max_pack_splits, n_kv_heads, n_packs); block = kAttnThreads.  One CTA per (split, kv head) reads the run's key
// blocks once for all of its segments; every row gets the bits of its segment's item run by attn_kvappend_kernel.
__global__ void __launch_bounds__(kAttnThreads, 1)
attn_kvappend_packed_kernel(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v,
                            const AttnParams p, const AttnPack* packs) {
  pdl_trigger();
  // the pack, item and page tables come from the memcpy at the start of the step: readable before the wait
  const AttnPack pk = packs[blockIdx.z];
  AttnItem it = p.items[pk.item0];
  const int split = blockIdx.x;
  if (split >= it.n_splits) return;
  it.q_count = pk.count;  // rows of the run: token t at q_tok0 + t, position q_pos0 + t
  attn_kvappend_cta<false, true>(tm_k, tm_v, p, it, split, blockIdx.y, 0, true, 0, 1, pk.item0);
}

// out[token, head, :] = sum_s O_s * 2^((m_s - M) c) / sum_s l_s * 2^((m_s - M) c)
// grid = (n_heads, n_tok_total); block = 128 (one thread per output dim).
struct AttnMergeParams {
  const float* ws_o;
  const float* ws_ml;
  const AttnItem* items;
  const int* tok_item;  // [n_tok] item index of each packed token
  __nv_bfloat16* out;   // [n_tok, n_heads * 128]
  int n_heads, n_kv_heads;
  float scale_log2;
};

constexpr int kMergeFast = 20;  // splits handled by the register-resident fast path (one wave: <= 18)

// Every thread fetches all (max, sum) pairs (broadcast loads) and its own column of all partial rows in ONE round
// of independent loads; weights are then computed redundantly per thread: no shared memory, no barrier.
template <int MAXS>
__device__ __forceinline__ float attn_merge_regs(const float* ws_ml, const float* o, size_t slot0, int rows, size_t stride,
                                                 int ns, float c) {
  float m[MAXS], l[MAXS], ov[MAXS];
#pragma unroll
  for (int s = 0; s < MAXS; ++s) {
    m[s] = -INFINITY, l[s] = 0.f, ov[s] = 0.f;
    if (s < ns) {
      const float2 ml = *reinterpret_cast<const float2*>(ws_ml + (slot0 + static_cast<size_t>(s) * rows) * 2);
      m[s] = ml.x, l[s] = ml.y;
      ov[s] = o[s * stride];
    }
  }
  float mx = -INFINITY;
#pragma unroll
  for (int s = 0; s < MAXS; ++s) mx = fmaxf(mx, m[s]);
  float den = 0.f, acc = 0.f;
#pragma unroll
  for (int s = 0; s < MAXS; ++s) {
    const float w = (m[s] == -INFINITY) ? 0.f : exp2f((m[s] - mx) * c);
    den += l[s] * w;
    acc += ov[s] * w;
  }
  return acc / den;
}

__global__ void __launch_bounds__(128) attn_merge_kernel(const AttnMergeParams p) {
  // one block per (head, token): thread d owns one output dim.
  __shared__ float s_m[160], s_w[160];
  __shared__ float s_den;
  const int head = blockIdx.x, tok = blockIdx.y, d = threadIdx.x;
  pdl_trigger();
  // the item tables were uploaded by the memcpy at the start of the step -> readable before the wait
  const AttnItem it = p.items[p.tok_item[tok]];
  const int G = p.n_heads / p.n_kv_heads;
  const int kvh = head / G, g = head % G;
  const int rows = it.q_count * G;
  const int r = (tok - it.q_tok0) * G + g;
  const float c = p.scale_log2;
  const size_t slot0 = static_cast<size_t>(it.ws_slot0) + static_cast<size_t>(kvh) * it.n_splits * rows + r;
  const int ns = it.n_splits;  // <= number of SMs
  const float* o = p.ws_o + slot0 * kAttnHD + d;
  const size_t stride = static_cast<size_t>(rows) * kAttnHD;
  __nv_bfloat16* dst = p.out + (static_cast<size_t>(tok) * p.n_heads + head) * kAttnHD + d;
  pdl_wait();
  if (ns <= 4) {   // many sequences per step (8 streams -> 2 splits each): keep the unrolled work proportional
    *dst = __float2bfloat16_rn(attn_merge_regs<4>(p.ws_ml, o, slot0, rows, stride, ns, c));
    return;
  }
  if (ns <= kMergeFast) {
    *dst = __float2bfloat16_rn(attn_merge_regs<kMergeFast>(p.ws_ml, o, slot0, rows, stride, ns, c));
    return;
  }
  // general path (many splits: one long sequence alone on the GPU with a tiny block budget)
  for (int s = d; s < ns; s += 128) {
    const float2 ml = *reinterpret_cast<const float2*>(p.ws_ml + (slot0 + static_cast<size_t>(s) * rows) * 2);
    s_m[s] = ml.x;
    s_w[s] = ml.y;
  }
  __syncthreads();
  float mx = -INFINITY;
  for (int s = 0; s < ns; ++s) mx = fmaxf(mx, s_m[s]);
  __syncthreads();
  for (int s = d; s < ns; s += 128) {
    const float m = s_m[s];
    const float w = (m == -INFINITY) ? 0.f : exp2f((m - mx) * c);
    s_m[s] = w;            // weight
    s_w[s] = s_w[s] * w;   // weighted row sum
  }
  __syncthreads();
  if (d == 0) {
    float den = 0.f;
    for (int s = 0; s < ns; ++s) den += s_w[s];
    s_den = den;
  }
  float acc = 0.f;
#pragma unroll 4
  for (int s = 0; s < ns; ++s) acc += o[s * stride] * s_m[s];
  __syncthreads();
  *dst = __float2bfloat16_rn(acc / s_den);
}

}  // namespace vlo
