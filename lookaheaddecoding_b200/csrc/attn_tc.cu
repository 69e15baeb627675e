// Lookahead attention, Hopper-native path (impl=2): TMA-staged K/V tiles, wgmma with register accumulators, the
// lookahead mask evaluated in registers, split-KV with an in-kernel merge through L2.
//
// Per CTA: one (head, 128-row query tile, KV split).  Warp roles (288 threads):
//   warps 0..7   two consumer warpgroups, 64 query rows each:
//                  S = Q K^T    (wgmma m64n128k16, Q and K from shared memory, both K-major)
//                  reference rounding -> mask bits -> exp2 -> P (model dtype) in registers, row max / sum by quad
//                  shuffles (the four threads of a quad hold one row)
//                  O += P V     (wgmma m64n128k16, P from registers, V from shared memory, MN-major)
//   warp 8       TMA producer: Q tile + a 3-deep ring of K/V tiles (128 kv rows x 128 d, SWIZZLE_128B); it also zeroes
//                the stale cache rows past kv_len + q_len of the last V tile (0 * NaN must not reach the MMA)
// Split merge: every split writes its fp32 partial rows to the scratch and takes a ticket on a per-(head, q tile)
// counter; the last CTA to arrive combines them in a fixed order.  The splits need not be co-resident, so impl 2 is a
// plain grid: a cluster of 4 one-SM CTAs must fit inside one GPC, and on an H100 SXM with 132 SMs only 30 such clusters
// fit at once -- the 32 heads of the decode step then ran in two rounds.
//
// Numerics follow attn_mma.cu / the reference (lade/models/modeling_llama.py:520-541); the mask is the
// same register predicate (common.cuh row_sees == modeling_llama.py:115-207).
//
// The reference-order variant (impl 3, REF = true) runs the same tiles and MMAs but rounds the probabilities the way
// the reference does (modeling_llama.py:530-541): p = model_dtype( exp(x - max_row) / sum_row ) with the max and the
// sum of the WHOLE row (all KV splits), normalised in fp32 BEFORE the rounding, then P.V with fp32 accumulation.  The
// online-softmax kernel has to round exp(x - max_so_far) before it knows the sum, which changes the last bit of about
// half of the outputs (DESIGN.md 6).  Knowing the whole row first means: every K/V tile of a split stays resident in
// shared memory (3 stages, so at most 3 KV tiles per split), S is recomputed by the tensor cores in each of the three
// passes (row max, row sum, P.V), and the splits of a head meet twice in the middle of the kernel (row maxima, then row
// sums, through an L2-resident table and a cluster barrier each).  It is an opt-in parity mode (impl = 3,
// `LookaheadEngine(attn_impl=3)`): slower, and bounded to kv_len + q_len <= 384 * n_splits.
#include "tc_common.cuh"

#include <cstdlib>
#include <mutex>
#include <type_traits>
#include <unordered_map>

namespace lade {

constexpr int TC_BM = 128;
constexpr int TC_BN = 128;
constexpr int TC_D = 128;
constexpr int TC_STAGES = 3;
constexpr int TC_CONSUMER_THREADS = 256;          // two warpgroups of 64 query rows
constexpr int TC_THREADS = TC_CONSUMER_THREADS + 32;
constexpr int TC_TILE_BYTES = 128 * 128 * 2;   // one [128 x 128] 16-bit tile = two [128 x 64] swizzle blocks
constexpr int TC_HALF_BYTES = TC_TILE_BYTES / 2;
constexpr int TC_SMEM_TILES = TC_TILE_BYTES * (1 + 2 * TC_STAGES);
constexpr int TC_SMEM_BYTES = TC_SMEM_TILES + 256 + 1024;   // tiles + mbarriers + slack to align the base to 1024 B
constexpr float TC_LOG2E = 1.4426950408889634f;
// Split merge: [counters: TC_MAX_COUNTERS ints, zero at rest][part_ml: (m, l) per split row][part_o: fp32 O per split
// row] at the start of the caller's scratch (lade_attn_scratch_bytes), the layout of the mma.sync kernel's merge.
constexpr int TC_MAX_COUNTERS = 16384;

// Optional per-CTA phase timestamps for profiling the kernel's own timeline: 16 slots per CTA, 0-7 hold %globaltimer
// (ns, one clock for the whole GPU, so CTAs on different SMs compare), 15 the SM the CTA ran on.
__device__ long long* g_attn_timing = nullptr;
__device__ __forceinline__ long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return (long long)t;
}
__device__ __forceinline__ int sm_id() {
  int s;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(s));
  return s;
}
#define TC_STAMP(slot, tid) do { if (tbuf && threadIdx.x == (tid)) tbuf[slot] = global_ns(); } while (0)
enum { TS_START = 0, TS_KFULL0 = 1, TS_SFULL0 = 2, TS_OFINAL = 3, TS_STAGED = 4, TS_TICKET = 5, TS_END = 7, TS_SMID = 15 };

// The model-dtype pair packed by Elem<ET>::pack2, back in fp32 (the rounded probabilities the row sum adds up).
template <typename ET> __device__ __forceinline__ float2 unpack2(uint32_t u);
template <> __device__ __forceinline__ float2 unpack2<__nv_bfloat16>(uint32_t u) {
  return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}
template <> __device__ __forceinline__ float2 unpack2<__half>(uint32_t u) {
  return __half22float2(*reinterpret_cast<__half2*>(&u));
}

// S[64 x 128] = Q[rows of warpgroup wg] . K^T of one stage.
template <typename ET>
__device__ __forceinline__ void qk_tile(float (&s)[64], uint32_t sQ_a, uint32_t sK_a, int wg) {
  wg_fence();
#pragma unroll
  for (int kb = 0; kb < 2; ++kb)
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t da = wg_desc(sQ_a + kb * TC_HALF_BYTES + wg * 8192 + k * 32, 16, 1024);
      const uint64_t db = wg_desc(sK_a + kb * TC_HALF_BYTES + k * 32, 16, 1024);
      wgmma_m64n128_ss<ET>(s, da, db, (kb | k) ? 1u : 0u);
    }
  wg_commit();
  wg_wait_all();
  wg_fence_regs(s);
}

// O[64 x 128] += P[64 x 128 kv] . V of one stage; p = the A fragments of the eight k16 steps (4 registers each).
template <typename ET>
__device__ __forceinline__ void pv_tile(float (&o)[64], const uint32_t (&p)[32], uint32_t sV_a) {
  wg_fence_regs(o);
  wg_fence();
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) wgmma_m64n128_rs_tb<ET>(o, p + 4 * kk, wg_desc(sV_a + kk * 2048, TC_HALF_BYTES, 1024));
  wg_commit();
  wg_wait_all();
  wg_fence_regs(o);
}

// Visibility of the 32 columns a thread holds in each of its two rows: word w of row rr covers tile columns [32w, 32w+32).
__device__ __forceinline__ void tile_mask(uint32_t (&mb)[2][4], const uint32_t* const (&mrow)[2], const int (&row)[2],
                                          int mask_words, int tile0, int kv_len, int q_len, int is_prefill) {
#pragma unroll
  for (int rr = 0; rr < 2; ++rr)
#pragma unroll
    for (int w = 0; w < 4; ++w)
      mb[rr][w] = (tile0 + 32 * w + 32 <= kv_len)
                      ? 0xffffffffu
                      : visible_bits32(mrow[rr], mask_words, tile0 + 32 * w, kv_len, q_len, is_prefill, row[rr]);
}
// accumulator element (i, e) of row half rr sits in tile column 8i + 2t + e: word i / 4, bit 8 (i % 4) + 2t + e
__device__ __forceinline__ bool vis(const uint32_t (&mb)[2][4], int rr, int i, int e, int t) {
  return (mb[rr][i >> 2] >> (8 * (i & 3) + 2 * t + e)) & 1u;
}

// ---- kernel ---------------------------------------------------------------------------------------------
// grid (n_splits, heads, q tiles); the n_splits CTAs of one (head, q tile) merge their split-KV partials through the
// scratch (impl 3 launches them as a thread-block cluster for its two mid-kernel exchanges).
template <typename ET, bool REF>
__global__ void __launch_bounds__(TC_THREADS, 1)
attn_fwd_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                   const __grid_constant__ CUtensorMap tmV, ET* __restrict__ out,
                   const uint32_t* __restrict__ rowmask, int mask_words, const int* __restrict__ meta, int q_pad,
                   int n_heads, int n_kv_heads, int n_splits, float inv_sqrt_d, int* __restrict__ counters,
                   float2* __restrict__ part_ml, float* __restrict__ part_o) {
  extern __shared__ unsigned char smem_raw[];
  const uint32_t raw_a = smem_u32(smem_raw);
  const uint32_t sQ_a = (raw_a + 1023u) & ~1023u;                  // SWIZZLE_128B tiles need 1024-byte alignment
  unsigned char* smem = smem_raw + (sQ_a - raw_a);
  const int split = blockIdx.x, h = blockIdx.y, mt = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  const int q_len = meta[LADE_M_Q_LEN];
  const int kv_len = meta[LADE_M_KV_LEN];
  const int is_prefill = meta[LADE_M_IS_PREFILL];
  const int T = kv_len + q_len;
  int Tm = T;
  if (is_prefill) Tm = min(T, kv_len + min(q_len, (mt + 1) * TC_BM));
  const int n_tiles = (Tm + TC_BN - 1) / TC_BN;
  // balanced partition: every split gets floor(n_tiles / n_splits) tiles, the first n_tiles % n_splits one more (the
  // LAST split holds the step columns -- masked softmax path, V-row zeroing -- and therefore never the extra tile)
  const int t_base = n_tiles / n_splits, t_rem = n_tiles - t_base * n_splits;
  const int n_active = n_tiles < n_splits ? n_tiles : n_splits;
  const bool active = split < n_active;
  const int tile_lo = split * t_base + (split < t_rem ? split : t_rem);
  const int my_tiles = active ? t_base + (split < t_rem ? 1 : 0) : 0;
  if (REF && t_base + (t_rem ? 1 : 0) > TC_STAGES) __trap();     // the caller's kv_bound was not a bound (host checks it)
  const int hk = h / (n_heads / n_kv_heads);
  const int HD = n_heads * TC_D;
  // split-major scratch tables: row r of this tile is row prow0 + r of split s's slab
  const long long slab = (long long)n_heads * gridDim.z * TC_BM;
  const long long prow0 = ((long long)h * gridDim.z + mt) * TC_BM;
  // a warpgroup whose 64 rows are all padding has nothing to compute
  const int n_wg = (mt * TC_BM + 64 < q_pad) ? 2 : 1;
  // the last tile of the launch may run past kv_len + q_len: its stale V rows are zeroed before P.V reads them
  const bool zero_last = active && (tile_lo + my_tiles) * TC_BN > T;
  long long* tbuf = g_attn_timing ? g_attn_timing + 16ll * ((blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) : nullptr;
  TC_STAMP(TS_START, 0);
  if (tbuf && threadIdx.x == 0) tbuf[TS_SMID] = sm_id();
  // programmatic dependent launch, producer side: a dependent grid may be scheduled as soon as SMs free up; it orders
  // itself with griddepcontrol.wait before it touches anything this grid writes
  griddep_launch_dependents();

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + TC_SMEM_TILES);
  // barrier slots: 0 q_full | 1.. k_full[S] | v_full[S] | stage_free[S] | v_zeroed
  const uint32_t bar0 = smem_u32(bars);
  auto BAR = [&](int i) { return bar0 + 8u * (uint32_t)i; };
  const int B_QFULL = 0, B_KFULL = 1, B_VFULL = 1 + TC_STAGES, B_FREE = 1 + 2 * TC_STAGES, B_VZERO = 1 + 3 * TC_STAGES;
  auto sK_a = [&](int s) { return sQ_a + (uint32_t)TC_TILE_BYTES * (1 + 2 * s); };
  auto sV_a = [&](int s) { return sQ_a + (uint32_t)TC_TILE_BYTES * (2 + 2 * s); };
  auto issue_tile = [&](int j) {
    const int s = j % TC_STAGES;
    const int row0 = (tile_lo + j) * TC_BN;
    mbar_expect_tx(BAR(B_KFULL + s), TC_TILE_BYTES);
    tma_load_3d(sK_a(s), &tmK, BAR(B_KFULL + s), 0, row0, hk);
    tma_load_3d(sK_a(s) + TC_HALF_BYTES, &tmK, BAR(B_KFULL + s), 64, row0, hk);
    mbar_expect_tx(BAR(B_VFULL + s), TC_TILE_BYTES);
    tma_load_3d(sV_a(s), &tmV, BAR(B_VFULL + s), 0, row0, hk);
    tma_load_3d(sV_a(s) + TC_HALF_BYTES, &tmV, BAR(B_VFULL + s), 64, row0, hk);
  };

  if (active && threadIdx.x == TC_CONSUMER_THREADS) {
    mbar_init(BAR(B_QFULL), 1);
    for (int s = 0; s < TC_STAGES; ++s) {
      mbar_init(BAR(B_KFULL + s), 1);
      mbar_init(BAR(B_VFULL + s), 1);
      mbar_init(BAR(B_FREE + s), 4 * n_wg);           // one arrival per consumer warp
    }
    mbar_init(BAR(B_VZERO), 1);
    fence_barrier_init();
    // Start the memory stream before anything else.  With programmatic dependent launch this CTA may already be
    // running while the producer of this step's Q and new K/V rows (lade_rope_append) is still in flight: cache tiles
    // entirely below kv_len were written by earlier steps and are fetched at once; Q and tiles touching rows >= kv_len
    // wait for the producer.
    const int n_pre = my_tiles < TC_STAGES ? my_tiles : TC_STAGES;
    int n_old = 0;                                   // leading tiles that hold only rows of earlier steps
    while (n_old < n_pre && (tile_lo + n_old + 1) * TC_BN <= kv_len) ++n_old;
    for (int j = 0; j < n_old; ++j) issue_tile(j);
    griddep_wait();
    mbar_expect_tx(BAR(B_QFULL), TC_TILE_BYTES);
    tma_load_3d(sQ_a, &tmQ, BAR(B_QFULL), 0, mt * TC_BM, h);
    tma_load_3d(sQ_a + TC_HALF_BYTES, &tmQ, BAR(B_QFULL), 64, mt * TC_BM, h);
    for (int j = n_old; j < n_pre; ++j) issue_tile(j);
  }
  __syncthreads();
  // Every thread that writes the scratch (split partials, (m, l) rows, the ticket counters) is ordered after the
  // predecessor grid here: under programmatic dependent launch that grid may be the previous attention launch, which
  // uses the same scratch.  In an active CTA the producer thread has already waited, so this returns at once.
  griddep_wait();

  // a consumer thread's share of its split's result: two rows (g and g + 8 of its warp's 16) x 32 of the 128 columns,
  // the unnormalised O (impl 2) or the normalised partial O (impl 3); kept in registers for the split merge
  const int wg = warp >> 2;
  const int g = lane >> 2, t = lane & 3;
  const int rl[2] = {wg * 64 + (warp & 3) * 16 + g, wg * 64 + (warp & 3) * 16 + g + 8};   // rows inside the tile
  const bool work = active && warp < 8 && wg < n_wg;
  float o[64];
  float m_row[2] = {-INFINITY, -INFINITY}, l_row[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;

  if (warp == 8) {
    // ================= TMA producer (tiles beyond the first STAGES; the rest was issued above) =================
    if (active) {
      if (lane == 0) {
        for (int j = TC_STAGES; j < my_tiles; ++j) {
          const int s = j % TC_STAGES;
          mbar_wait(BAR(B_FREE + s), ((j / TC_STAGES) - 1) & 1);
          issue_tile(j);
        }
      }
      __syncwarp();
      if (zero_last) {
        const int j = my_tiles - 1, s = j % TC_STAGES;
        const int r0 = T - (tile_lo + j) * TC_BN;      // first stale row of the tile
        mbar_wait(BAR(B_VFULL + s), (j / TC_STAGES) & 1);
        unsigned char* pV = smem + TC_TILE_BYTES * (2 + 2 * s);
        const uint4 z = make_uint4(0, 0, 0, 0);
        for (int c = r0 * 8 + lane; c < TC_BN * 8; c += 32) {      // whole 128-byte rows: the swizzle does not matter
          const int r = c >> 3, cc = c & 7;
          *reinterpret_cast<uint4*>(pV + r * 128 + cc * 16) = z;
          *reinterpret_cast<uint4*>(pV + TC_HALF_BYTES + r * 128 + cc * 16) = z;
        }
        fence_proxy_async();                          // the zeros -> visible to the tensor core's async proxy
        __syncwarp();
        if (lane == 0) mbar_arrive(BAR(B_VZERO));
      }
    }
    if (REF) {                                        // meet the cluster at the row-max and row-sum exchanges
      cluster_arrive(); cluster_wait();
      cluster_arrive(); cluster_wait();
    }
  } else {
    const int row[2] = {mt * TC_BM + rl[0], mt * TC_BM + rl[1]};   // step-local rows
    const uint32_t* const mrow[2] = {
        (row[0] < q_pad && !is_prefill && rowmask != nullptr) ? rowmask + (long long)row[0] * mask_words : nullptr,
        (row[1] < q_pad && !is_prefill && rowmask != nullptr) ? rowmask + (long long)row[1] * mask_words : nullptr};
    auto wait_v = [&](int j) {
      const int s = j % TC_STAGES;
      mbar_wait(BAR(B_VFULL + s), (j / TC_STAGES) & 1);
      if (zero_last && j == my_tiles - 1) mbar_wait(BAR(B_VZERO), 0);
    };
    if (work) mbar_wait(BAR(B_QFULL), 0);
    if (!REF) {
      // ================= online softmax: one pass over the split's tiles =================
      for (int j = 0; work && j < my_tiles; ++j) {
        const int s = j % TC_STAGES;
        const int tile0 = (tile_lo + j) * TC_BN;
        mbar_wait(BAR(B_KFULL + s), (j / TC_STAGES) & 1);
        if (j == 0) TC_STAMP(TS_KFULL0, 0);
        float sc[64];
        qk_tile<ET>(sc, sQ_a, sK_a(s), wg);
        if (j == 0) TC_STAMP(TS_SFULL0, 0);
        uint32_t mb[2][4];
        tile_mask(mb, mrow, row, mask_words, tile0, kv_len, q_len, is_prefill);
        // row max of the raw scores; bf16 rounding and the positive scale are monotone, so round the max once
        float off[2];
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          float mx = -INFINITY;
#pragma unroll
          for (int i = 0; i < 16; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) mx = fmaxf(mx, vis(mb, rr, i, e, t) ? sc[4 * i + 2 * rr + e] : -INFINITY);
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
          const float mtile = mx == -INFINITY ? -INFINITY : round_to<ET>(round_to<ET>(mx) * inv_sqrt_d);
          if (mtile > m_row[rr]) {                    // the running max grew: rescale what was accumulated so far
            const float scale = m_row[rr] == -INFINITY ? 1.f : exp2f((m_row[rr] - mtile) * TC_LOG2E);
            l_row[rr] *= scale;
#pragma unroll
            for (int i = 0; i < 16; ++i) { o[4 * i + 2 * rr] *= scale; o[4 * i + 2 * rr + 1] *= scale; }
            m_row[rr] = mtile;
          }
          off[rr] = m_row[rr] == -INFINITY ? 0.f : m_row[rr] * TC_LOG2E;
        }
        // P = exp2(score - max) in the model dtype, straight into the A fragments of P.V; the row sum adds the ROUNDED
        // probabilities (the normaliser of exactly what the MMA multiplies)
        uint32_t pa[32];
#pragma unroll
        for (int i = 0; i < 16; ++i)
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            float r0, r1;
            round_scale_round2<ET>(sc[4 * i + 2 * rr], sc[4 * i + 2 * rr + 1], inv_sqrt_d, r0, r1);
            const float p0 = vis(mb, rr, i, 0, t) ? ex2_approx(r0 * TC_LOG2E - off[rr]) : 0.f;
            const float p1 = vis(mb, rr, i, 1, t) ? ex2_approx(r1 * TC_LOG2E - off[rr]) : 0.f;
            const uint32_t pk = Elem<ET>::pack2(p0, p1);
            const float2 pr = unpack2<ET>(pk);
            l_row[rr] += pr.x + pr.y;
            pa[4 * (i >> 1) + 2 * (i & 1) + rr] = pk;
          }
        wait_v(j);
        pv_tile<ET>(o, pa, sV_a(s));
        __syncwarp();
        if (lane == 0) mbar_arrive(BAR(B_FREE + s));
      }
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        l_row[rr] += __shfl_xor_sync(0xffffffffu, l_row[rr], 1);
        l_row[rr] += __shfl_xor_sync(0xffffffffu, l_row[rr], 2);
      }
    } else {
      // ================= reference order: row max, row sum, then P.V, S recomputed in each pass =================
      float sc[64];
      uint32_t mb[2][4];
      // ---- pass A: the row maximum of the split
      float mx[2] = {-INFINITY, -INFINITY};
      for (int j = 0; work && j < my_tiles; ++j) {
        mbar_wait(BAR(B_KFULL + j), 0);
        qk_tile<ET>(sc, sQ_a, sK_a(j), wg);
        tile_mask(mb, mrow, row, mask_words, (tile_lo + j) * TC_BN, kv_len, q_len, is_prefill);
#pragma unroll
        for (int rr = 0; rr < 2; ++rr)
#pragma unroll
          for (int i = 0; i < 16; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) mx[rr] = fmaxf(mx[rr], vis(mb, rr, i, e, t) ? sc[4 * i + 2 * rr + e] : -INFINITY);
      }
      if (work) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 1));
          mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 2));
          const float m_split = mx[rr] == -INFINITY ? -INFINITY : round_to<ET>(round_to<ET>(mx[rr]) * inv_sqrt_d);
          if (t == 0) part_ml[split * slab + prow0 + rl[rr]].x = m_split;
        }
      }
      cluster_arrive(); cluster_wait();
      float m_ref[2] = {0.f, 0.f};
      if (work) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          float m_all = -INFINITY;
          for (int sp = 0; sp < n_active; ++sp)
            m_all = fmaxf(m_all, ld_global_f2(part_ml + sp * slab + prow0 + rl[rr]).x);
          m_ref[rr] = (m_all == -INFINITY) ? 0.f : m_all;   // x - max is exact in fp32 (both are model-dtype values)
        }
      }
      // e = exp(x - max) in fp32 of tile j (S recomputed from the resident K tile)
      auto exps = [&](int j) {
        qk_tile<ET>(sc, sQ_a, sK_a(j), wg);
        tile_mask(mb, mrow, row, mask_words, (tile_lo + j) * TC_BN, kv_len, q_len, is_prefill);
#pragma unroll
        for (int i = 0; i < 16; ++i)
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            float r0, r1;
            round_scale_round2<ET>(sc[4 * i + 2 * rr], sc[4 * i + 2 * rr + 1], inv_sqrt_d, r0, r1);
            sc[4 * i + 2 * rr] = vis(mb, rr, i, 0, t) ? ex2_approx((r0 - m_ref[rr]) * TC_LOG2E) : 0.f;
            sc[4 * i + 2 * rr + 1] = vis(mb, rr, i, 1, t) ? ex2_approx((r1 - m_ref[rr]) * TC_LOG2E) : 0.f;
          }
      };
      // ---- pass B: the row sum of the split
      float l_part[2] = {0.f, 0.f};
      for (int j = 0; work && j < my_tiles; ++j) {
        exps(j);
#pragma unroll
        for (int rr = 0; rr < 2; ++rr)
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            l_part[rr] += sc[4 * i + 2 * rr];
            l_part[rr] += sc[4 * i + 2 * rr + 1];
          }
      }
      if (work) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          l_part[rr] += __shfl_xor_sync(0xffffffffu, l_part[rr], 1);
          l_part[rr] += __shfl_xor_sync(0xffffffffu, l_part[rr], 2);
          if (t == 0) part_ml[split * slab + prow0 + rl[rr]].y = l_part[rr];
        }
      }
      cluster_arrive(); cluster_wait();
      float l_all[2] = {0.f, 0.f};
      if (work) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr)
          for (int sp = 0; sp < n_active; ++sp) l_all[rr] += ld_global_f2(part_ml + sp * slab + prow0 + rl[rr]).y;
      }
      // ---- pass C: p = model_dtype(e / sum) -> P.V, tile by tile
      for (int j = 0; work && j < my_tiles; ++j) {
        exps(j);
        uint32_t pa[32];
#pragma unroll
        for (int i = 0; i < 16; ++i)
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const float p0 = l_all[rr] > 0.f ? __fdiv_rn(sc[4 * i + 2 * rr], l_all[rr]) : 0.f;
            const float p1 = l_all[rr] > 0.f ? __fdiv_rn(sc[4 * i + 2 * rr + 1], l_all[rr]) : 0.f;
            pa[4 * (i >> 1) + 2 * (i & 1) + rr] = Elem<ET>::pack2(p0, p1);
          }
        wait_v(j);
        pv_tile<ET>(o, pa, sV_a(j));
      }
    }
    TC_STAMP(TS_OFINAL, 0);
    if (work && n_splits == 1) {
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        if (row[rr] >= q_pad) continue;
        const float inv = REF ? 1.f : (l_row[rr] > 0.f ? 1.f / l_row[rr] : 0.f);
        uint32_t* dst = reinterpret_cast<uint32_t*>(out + (long long)row[rr] * HD + h * TC_D + 2 * t);
#pragma unroll
        for (int i = 0; i < 16; ++i) dst[4 * i] = Elem<ET>::pack2(o[4 * i + 2 * rr] * inv, o[4 * i + 2 * rr + 1] * inv);
      }
    }
  }
  if (n_splits == 1) { TC_STAMP(TS_END, 0); return; }
  if (!active) return;                                // a split without tiles takes no part in the merge

  // ---- split merge through L2, by the CTA that arrives last ----
  // Every split stores its partial rows (fp32 O; impl 2 also (m, l)) in the scratch, fences, and takes a ticket on the
  // (head, q tile) counter; the CTA that draws the last ticket combines all of them and puts the counter back to 0.
  // Row r of the tile is combined in a fixed order: its owning split r / per (per = ceil(rows / n_active)) first, then
  // the others in ascending split order, every step rounded as written (no contraction can move a bit):
  //   impl 2:  w_s = 2^(m_s - m),  out = (sum_s w_s O_s) * (1 / sum_s w_s l_s)        impl 3:  out = sum_s O_s
  // A single active split is its own last CTA and merges from registers.
  const int rows_valid = min(TC_BM, q_pad - mt * TC_BM);
  const int per = (rows_valid + n_active - 1) / n_active;
  int* const counter = counters + h * gridDim.z + mt;
  if (n_active > 1) {
    __shared__ int s_last;
    if (work) {
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        if (rl[rr] >= rows_valid) continue;
        float2* po = reinterpret_cast<float2*>(part_o + (split * slab + prow0 + rl[rr]) * TC_D + 2 * t);
#pragma unroll
        for (int i = 0; i < 16; ++i) po[4 * i] = make_float2(o[4 * i + 2 * rr], o[4 * i + 2 * rr + 1]);
        if (!REF && t == 0) part_ml[split * slab + prow0 + rl[rr]] = make_float2(m_row[rr], l_row[rr]);
      }
    }
    TC_STAMP(TS_STAGED, 0);
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(counter, 1) == n_active - 1;
    __syncthreads();
    TC_STAMP(TS_TICKET, 0);
    if (!s_last) return;
    __threadfence();
    if (threadIdx.x == 0) *counter = 0;             // every split has drawn its ticket: ready for the next launch
  }
  if (work && n_active == 1) {                        // the partial is the result: it never left the registers
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      if (rl[rr] >= rows_valid) continue;
      float wgt = 1.f, inv = 1.f;
      if (!REF) {
        wgt = (m_row[rr] == -INFINITY) ? 0.f : exp2f((m_row[rr] - m_row[rr]) * TC_LOG2E);
        const float lsum = __fmul_rn(l_row[rr], wgt);
        inv = lsum > 0.f ? 1.f / lsum : 0.f;
      }
      uint32_t* dst = reinterpret_cast<uint32_t*>(out + (long long)(mt * TC_BM + rl[rr]) * HD + h * TC_D + 2 * t);
#pragma unroll
      for (int i = 0; i < 16; ++i)
        dst[4 * i] = Elem<ET>::pack2(__fmul_rn(__fmul_rn(o[4 * i + 2 * rr], wgt), inv),
                                     __fmul_rn(__fmul_rn(o[4 * i + 2 * rr + 1], wgt), inv));
    }
  } else if (work) {
    // Both rows of the thread advance together and every split's rows are loaded before they are used, so the merge
    // costs about n_active + 1 L2 round trips.  The CTA's own partial is read back from L2 like the others.
    bool valid[2];
    int own[2];
    const float2* pml[2];
    const float2* po[2];
    float mmax[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      valid[rr] = rl[rr] < rows_valid;
      own[rr] = rl[rr] / per;
      pml[rr] = part_ml + prow0 + rl[rr];
      po[rr] = reinterpret_cast<const float2*>(part_o + (prow0 + rl[rr]) * TC_D + 2 * t);
      mmax[rr] = -INFINITY;                          // max over the splits: exact, so its order does not matter
      if (!REF && valid[rr]) {
        float mx[8];
#pragma unroll
        for (int s = 0; s < 8; ++s) mx[s] = s < n_active ? __ldcg(pml[rr] + s * slab).x : -INFINITY;
#pragma unroll
        for (int s = 0; s < 8; ++s) mmax[rr] = fmaxf(mmax[rr], mx[s]);
      }
    }
    float acc[2][32], lsum[2] = {0.f, 0.f};
    for (int k = 0; k < n_active; ++k) {
      float2 x[2][16], ml[2];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {               // the owning split first, then the others in ascending order
        const int s = k == 0 ? own[rr] : (k - 1 < own[rr] ? k - 1 : k);
        if (!valid[rr]) continue;
        if (!REF) ml[rr] = __ldcg(pml[rr] + s * slab);
#pragma unroll
        for (int i = 0; i < 16; ++i) x[rr][i] = __ldcg(po[rr] + s * slab * (TC_D / 2) + 4 * i);
      }
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        if (!valid[rr]) continue;
        if (!REF) {
          const float wgt = (ml[rr].x == -INFINITY) ? 0.f : exp2f((ml[rr].x - mmax[rr]) * TC_LOG2E);
          lsum[rr] = k == 0 ? __fmul_rn(ml[rr].y, wgt) : __fmaf_rn(ml[rr].y, wgt, lsum[rr]);
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            acc[rr][2 * i] = k == 0 ? __fmul_rn(x[rr][i].x, wgt) : __fmaf_rn(x[rr][i].x, wgt, acc[rr][2 * i]);
            acc[rr][2 * i + 1] = k == 0 ? __fmul_rn(x[rr][i].y, wgt) : __fmaf_rn(x[rr][i].y, wgt, acc[rr][2 * i + 1]);
          }
        } else {
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            acc[rr][2 * i] = k == 0 ? x[rr][i].x : __fadd_rn(acc[rr][2 * i], x[rr][i].x);
            acc[rr][2 * i + 1] = k == 0 ? x[rr][i].y : __fadd_rn(acc[rr][2 * i + 1], x[rr][i].y);
          }
        }
      }
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      if (!valid[rr]) continue;
      const float inv = REF ? 1.f : (lsum[rr] > 0.f ? 1.f / lsum[rr] : 0.f);
      uint32_t* dst = reinterpret_cast<uint32_t*>(out + (long long)(mt * TC_BM + rl[rr]) * HD + h * TC_D + 2 * t);
#pragma unroll
      for (int i = 0; i < 16; ++i)
        dst[4 * i] = Elem<ET>::pack2(__fmul_rn(acc[rr][2 * i], inv), __fmul_rn(acc[rr][2 * i + 1], inv));
    }
  }
  TC_STAMP(TS_END, 0);
}

int attn_tc_set_timing_buffer(void* dev_ptr) {
  long long* p = reinterpret_cast<long long*>(dev_ptr);
  cudaError_t e = cudaMemcpyToSymbol(g_attn_timing, &p, sizeof(p));
  if (e != cudaSuccess) { set_cuda_error(e, "cudaMemcpyToSymbol(g_attn_timing)"); return LADE_ECUDA; }
  return LADE_OK;
}

// ---- host: tensor maps ----------------------------------------------------------------------------------
EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

struct MapKey {
  const void* ptr; int rows; int heads;
  bool operator==(const MapKey& o) const { return ptr == o.ptr && rows == o.rows && heads == o.heads; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    return std::hash<const void*>()(k.ptr) ^ (std::hash<int>()(k.rows) * 31) ^ (std::hash<int>()(k.heads) * 131);
  }
};

// [heads][rows][128] bf16, box = 64 d x 128 rows x 1 head, SWIZZLE_128B; out-of-range rows are zero filled
static int get_tensor_map(const void* ptr, int rows, int heads, CUtensorMap* out) {
  static std::mutex mu;
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  std::lock_guard<std::mutex> lock(mu);
  MapKey key{ptr, rows, heads};
  auto it = cache.find(key);
  if (it != cache.end()) { *out = it->second; return LADE_OK; }
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return LADE_EUNSUPPORTED;
  CUtensorMap tm;
  const cuuint64_t dims[3] = {(cuuint64_t)TC_D, (cuuint64_t)rows, (cuuint64_t)heads};
  const cuuint64_t strides[2] = {(cuuint64_t)TC_D * 2, (cuuint64_t)rows * TC_D * 2};
  const cuuint32_t box[3] = {64, 128, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return LADE_ECUDA;
  if (cache.size() > 4096) cache.clear();
  cache.emplace(key, tm);
  *out = tm;
  return LADE_OK;
}

static int g_pdl_override = -1;      // lade_debug_attn_pdl: -1 = environment (LADE_PDL), 0 / 1 = forced
int attn_tc_set_pdl(int v) { g_pdl_override = v < 0 ? -1 : (v ? 1 : 0); return LADE_OK; }

static bool pdl_enabled() {
  if (g_pdl_override >= 0) return g_pdl_override != 0;
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("LADE_PDL");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v != 0;
}

// One launch of attn_fwd_tc_kernel<ET, REF>: grid (n_splits, heads, q tiles).  The reference-order variant meets its
// sibling splits twice in the middle of the kernel, so the splits of a (head, q tile) form a cluster (co-resident);
// impl 2 needs no co-residency and is launched as a plain grid.
template <typename ET, bool REF>
static int launch_tc(cudaStream_t stream, const void* q, const void* k_cache, const void* v_cache, void* out,
                     const uint32_t* rowmask, int mask_words, const int32_t* meta, void* scratch, int q_pad, int n_heads,
                     int n_kv_heads, int head_dim, int kv_capacity, int n_splits) {
  const int q_tiles = (q_pad + TC_BM - 1) / TC_BM;
  if ((long long)n_heads * q_tiles > TC_MAX_COUNTERS) return LADE_EUNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(q) & 15) || (reinterpret_cast<uintptr_t>(k_cache) & 15) ||
      (reinterpret_cast<uintptr_t>(v_cache) & 15))
    return LADE_EINVAL;
  CUtensorMap tmQ, tmK, tmV;
  int rc;
  if ((rc = get_tensor_map(q, q_pad, n_heads, &tmQ)) != LADE_OK) return rc;
  if ((rc = get_tensor_map(k_cache, kv_capacity, n_kv_heads, &tmK)) != LADE_OK) return rc;
  if ((rc = get_tensor_map(v_cache, kv_capacity, n_kv_heads, &tmV)) != LADE_OK) return rc;
  static unsigned long long attr_devs = 0;   // the attribute is per device (context): one bit per ordinal
  int cur_dev = 0;
  LADE_CUDA_CHECK(cudaGetDevice(&cur_dev));
  if (!((attr_devs >> (cur_dev & 63)) & 1ull)) {
    LADE_CUDA_CHECK(cudaFuncSetAttribute(attn_fwd_tc_kernel<ET, REF>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_BYTES));
    attr_devs |= 1ull << (cur_dev & 63);
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(n_splits, n_heads, q_tiles);
  cfg.blockDim = dim3(TC_THREADS);
  cfg.dynamicSmemBytes = TC_SMEM_BYTES;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int n_attr = 0;
  // programmatic dependent launch: the grid may start while its stream predecessor (lade_rope_append, which signals
  // griddepcontrol.launch_dependents at entry) is still running; the kernel orders itself with griddepcontrol.wait
  if (pdl_enabled()) {
    attr[n_attr].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n_attr++].val.programmaticStreamSerializationAllowed = 1;
  }
  if (REF) {
    attr[n_attr].id = cudaLaunchAttributeClusterDimension;
    attr[n_attr].val.clusterDim.x = n_splits;
    attr[n_attr].val.clusterDim.y = 1;
    attr[n_attr++].val.clusterDim.z = 1;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n_attr;
  const float inv_sqrt_d = 1.0f / sqrtf((float)head_dim);
  // scratch (lade_attn_scratch_bytes): [counters][part_ml][part_o] with n_splits * n_heads * q_tiles * 128 rows per table
  int* counters = reinterpret_cast<int*>(scratch);
  float2* part_ml = reinterpret_cast<float2*>(counters + TC_MAX_COUNTERS);
  float* part_o = reinterpret_cast<float*>(part_ml + (size_t)n_splits * n_heads * q_tiles * TC_BM);
  cudaError_t e = cudaLaunchKernelEx(&cfg, attn_fwd_tc_kernel<ET, REF>, tmQ, tmK, tmV, (ET*)out, rowmask, mask_words, meta,
                                     q_pad, n_heads, n_kv_heads, n_splits, inv_sqrt_d, counters, part_ml, part_o);
  if (e != cudaSuccess) { set_cuda_error(e, "cudaLaunchKernelEx(attn_fwd_tc_kernel)"); return LADE_ECUDA; }
  return LADE_OK;
}

template <typename ET>
static int attn_fwd_tc_launch_t(cudaStream_t stream, const void* q, const void* k_cache, const void* v_cache, void* out,
                                const uint32_t* rowmask, int mask_words, const int32_t* meta, void* scratch, int q_pad,
                                int n_heads, int n_kv_heads, int head_dim, int kv_capacity, int kv_bound, int n_splits) {
  (void)kv_bound;
  if (head_dim != TC_D) return LADE_EUNSUPPORTED;
  if (n_splits > 8) n_splits = 8;   // the split count shapes the numerics: same clamp as the cluster-launched impl 3
  return launch_tc<ET, false>(stream, q, k_cache, v_cache, out, rowmask, mask_words, meta, scratch, q_pad, n_heads,
                              n_kv_heads, head_dim, kv_capacity, n_splits);
}

int attn_fwd_tc_launch(cudaStream_t stream, const void* q, const void* k_cache, const void* v_cache, void* out,
                       const uint32_t* rowmask, int mask_words, const int32_t* meta, void* scratch, int q_pad, int n_heads,
                       int n_kv_heads, int head_dim, int kv_capacity, int kv_bound, int n_splits, int is_f16) {
  if (is_f16)
    return attn_fwd_tc_launch_t<__half>(stream, q, k_cache, v_cache, out, rowmask, mask_words, meta, scratch, q_pad, n_heads,
                                        n_kv_heads, head_dim, kv_capacity, kv_bound, n_splits);
  return attn_fwd_tc_launch_t<__nv_bfloat16>(stream, q, k_cache, v_cache, out, rowmask, mask_words, meta, scratch, q_pad,
                                             n_heads, n_kv_heads, head_dim, kv_capacity, kv_bound, n_splits);
}

// impl 3: the reference-order variant.  kv_bound must bound kv_len + q_len of this call (every K/V tile of a split stays
// resident in shared memory: at most 3 per split); the kernel traps if it does not.
template <typename ET>
static int attn_fwd_tc_exact_launch_t(cudaStream_t stream, const void* q, const void* k_cache, const void* v_cache, void* out,
                                      const uint32_t* rowmask, int mask_words, const int32_t* meta, void* scratch, int q_pad,
                                      int n_heads, int n_kv_heads, int head_dim, int kv_capacity, int kv_bound, int n_splits) {
  if (head_dim != TC_D) return LADE_EUNSUPPORTED;
  if (n_splits > 8) n_splits = 8;
  if (kv_bound < 1 || (kv_bound + TC_BN - 1) / TC_BN > TC_STAGES * n_splits) {
    set_error_string("lade_attn_fwd impl 3: kv_bound exceeds 384 * n_splits (every K/V tile of a split must stay in shared memory)");
    return LADE_EUNSUPPORTED;
  }
  return launch_tc<ET, true>(stream, q, k_cache, v_cache, out, rowmask, mask_words, meta, scratch, q_pad, n_heads,
                             n_kv_heads, head_dim, kv_capacity, n_splits);
}

int attn_fwd_tc_exact_launch(cudaStream_t stream, const void* q, const void* k_cache, const void* v_cache, void* out,
                             const uint32_t* rowmask, int mask_words, const int32_t* meta, void* scratch, int q_pad, int n_heads,
                             int n_kv_heads, int head_dim, int kv_capacity, int kv_bound, int n_splits, int is_f16) {
  if (is_f16)
    return attn_fwd_tc_exact_launch_t<__half>(stream, q, k_cache, v_cache, out, rowmask, mask_words, meta, scratch, q_pad,
                                              n_heads, n_kv_heads, head_dim, kv_capacity, kv_bound, n_splits);
  return attn_fwd_tc_exact_launch_t<__nv_bfloat16>(stream, q, k_cache, v_cache, out, rowmask, mask_words, meta, scratch, q_pad,
                                                   n_heads, n_kv_heads, head_dim, kv_capacity, kv_bound, n_splits);
}

}  // namespace lade
