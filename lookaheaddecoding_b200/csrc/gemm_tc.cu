// Weight-streaming projection GEMM for the lookahead step on sm_90a (wgmma + TMA).
//
//   C[M, N] = A[M, K] · W[N, K]^T      bf16 in / bf16 out, fp32 accumulation in registers
//
// Replaces the nn.Linear calls of the reference decoder layer on the lookahead step
// (lade/models/modeling_llama.py:447-449 q/k/v_proj, :541 o_proj, :378 gate/up/down_proj, :1608 lm_head)
// for the step's row count M <= 128 (W*(N-1) window rows + guess rows).  With so few rows the GEMM is a pure
// stream of the weight matrix out of HBM, so the design goal is "every SM pulls weights all the time":
//
//   * one CTA per (N tile, K split); the tile width BN (32..256) and the K split (1/2/4/8) are picked per
//     shape so that the CTA count lands just under the SM count (a single full wave);
//   * warp 8 = TMA producer (A k-block [128 x 64] from L2, W k-block [BN x 64] from HBM, SWIZZLE_128B) into a
//     4-11 stage mbarrier ring; warps 0-7 = two consumer warpgroups, 64 rows of A each (the second one idles when
//     M <= 64), wgmma m64n32k16 x BN / 32 per k16 step, accumulator [64 x BN] fp32 in registers;
//   * K splits of one N tile form a thread-block cluster; their fp32 partial tiles are staged in shared memory
//     and summed over distributed shared memory (no global scratch, no atomics, deterministic order).
//
// Rows >= M of the A box are zero-filled by TMA; W rows >= N likewise, so ragged tiles need no special casing
// beyond the store guards.
#include "tc_common.cuh"

#include <mutex>
#include <unordered_map>

namespace lade {

constexpr int GM_THREADS = 288;          // two consumer warpgroups + one producer warp
constexpr int GM_PRODUCER = 256;         // the producer thread
constexpr int GM_BK = 64;                   // one SWIZZLE_128B atom of bf16 along K
constexpr int GM_A_BYTES = 128 * GM_BK * 2; // 16 KB
constexpr int GM_MAX_STAGES = 11;
constexpr int GM_SMEM_LIMIT = 227 * 1024;
constexpr int GM_BAR_BYTES = 8 * (2 * GM_MAX_STAGES + 2);

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1) : "memory");
}

// Optional per-CTA phase timestamps (%globaltimer, ns): 8 int64 per CTA, 4 launches round-robin (lade_debug_gemm_timing).
__device__ long long* g_gemm_timing = nullptr;
__device__ __forceinline__ long long globaltimer_ns() {
  long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
#define GM_STAMP(slot, tid) do { if (tbuf && threadIdx.x == (tid)) tbuf[slot] = globaltimer_ns(); } while (0)

// Sum the SK fp32 partial tiles of one N tile over distributed shared memory.  The remote loads of a batch are all
// issued before the first use so their (long) latencies overlap.
template <int SK>
__device__ __forceinline__ void reduce_splits(__nv_bfloat16* __restrict__ C, uint32_t smem_base, int BN, int M, int N, int ldc,
                                              int n0, int y) {
  constexpr int ITEMS = 16 / SK;                 // float4 items per thread per batch: 16 loads in flight
  const int rows_per = 128 / SK;
  const int r0 = y * rows_per;
  const int c4n = BN >> 2;
  const int total = rows_per * c4n;
  uint32_t peer_base[SK];
#pragma unroll
  for (int p = 0; p < SK; ++p) peer_base[p] = dsmem_addr(smem_base, (uint32_t)p);
  for (int i0 = threadIdx.x; i0 < total; i0 += ITEMS * GM_THREADS) {
    float4 v[ITEMS][SK];
#pragma unroll
    for (int it = 0; it < ITEMS; ++it) {
      const int i = i0 + it * GM_THREADS;
      if (i < total) {
        const int r = r0 + i / c4n;
        const int c4 = i - (i / c4n) * c4n;
        const uint32_t off = (uint32_t)((r * (BN + 4) + c4 * 4) * 4);
#pragma unroll
        for (int p = 0; p < SK; ++p) v[it][p] = ld_dsmem_f4(peer_base[p] + off);
      }
    }
#pragma unroll
    for (int it = 0; it < ITEMS; ++it) {
      const int i = i0 + it * GM_THREADS;
      if (i < total) {
        const int r = r0 + i / c4n;
        const int c4 = i - (i / c4n) * c4n;
        float4 acc = v[it][0];
#pragma unroll
        for (int p = 1; p < SK; ++p) { acc.x += v[it][p].x; acc.y += v[it][p].y; acc.z += v[it][p].z; acc.w += v[it][p].w; }
        const int n = n0 + c4 * 4;
        if (r < M && n < N) {
          uint2 o;
          o.x = pack2_bf16(acc.x, acc.y);
          o.y = pack2_bf16(acc.z, acc.w);
          *reinterpret_cast<uint2*>(C + (size_t)r * ldc + n) = o;
        }
      }
    }
  }
}

__global__ void __launch_bounds__(GM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
               __nv_bfloat16* __restrict__ C, int M, int N, int ldc, int kb_per_split, int BN, int stages, int split_k,
               int prefill, int launch_id) {
  long long* tbuf = g_gemm_timing ? g_gemm_timing + 8ll * ((launch_id & 3) * 1024 + blockIdx.y * gridDim.x + blockIdx.x) : nullptr;
  GM_STAMP(0, GM_PRODUCER);
  extern __shared__ uint8_t smem_raw[];
  // ring stage = [128 x 64] activations | [BN x 64] weights, one full / one empty mbarrier per stage; the base is
  // aligned to 1024 bytes by hand (SWIZZLE_128B), the launch reserves the slack
  const uint32_t raw_a = smem_u32(smem_raw);
  const uint32_t smem_base = (raw_a + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (smem_base - raw_a);
  const int stage_bytes = GM_A_BYTES + BN * 128;
  const uint32_t bars = smem_base + stages * stage_bytes;
  auto FULL = [&](int s) { return bars + 8u * s; };
  auto EMPTY = [&](int s) { return bars + 8u * (GM_MAX_STAGES + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n0 = blockIdx.x * BN;
  const int kb0 = blockIdx.y * kb_per_split;
  const int n_wg = M > 64 ? 2 : 1;                 // warpgroups with rows of A to multiply

  auto issue = [&](int kb) {
    const int s = kb % stages;
    const uint32_t sa = smem_base + s * stage_bytes;
    mbar_expect_tx(FULL(s), (uint32_t)stage_bytes);
    tma_load_2d(sa + GM_A_BYTES, &tmW, FULL(s), (kb0 + kb) * GM_BK, n0);
    tma_load_2d(sa, &tmA, FULL(s), (kb0 + kb) * GM_BK, 0);
  };

  if (tid == GM_PRODUCER) {
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmA);
    for (int s = 0; s < stages; ++s) { mbar_init(FULL(s), 1); mbar_init(EMPTY(s), 4 * n_wg); }
    fence_barrier_init();
    // nothing has to be waited for to fill the ring: do it before the CTA has finished setting up
    if (prefill) for (int kb = 0; kb < stages; ++kb) issue(kb);
  }
  __syncthreads();
  GM_STAMP(1, GM_PRODUCER);

  const int wg = warp >> 2;
  const int g = lane >> 2, t = lane & 3;
  const int row0 = wg * 64 + (warp & 3) * 16 + g;   // this thread's rows: row0 and row0 + 8
  float acc[8][16];
#pragma unroll
  for (int c = 0; c < 8; ++c)
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[c][i] = 0.f;

  if (warp == 8) {
    if (lane == 0) {
      for (int kb = prefill ? stages : 0; kb < kb_per_split; ++kb) {
        if (kb >= stages) mbar_wait(EMPTY(kb % stages), ((kb / stages) - 1) & 1);
        issue(kb);
      }
    }
    __syncwarp();
  } else if (wg < n_wg) {
    for (int kb = 0; kb < kb_per_split; ++kb) {
      const int s = kb % stages;
      mbar_wait(FULL(s), (kb / stages) & 1);
      if (kb == 0) GM_STAMP(2, 0);
      const uint32_t sa = smem_base + s * stage_bytes;
#pragma unroll
      for (int c = 0; c < 8; ++c) wg_fence_regs(acc[c]);
      wg_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t da = wg_desc(sa + wg * 8192 + k * 32, 16, 1024);
#pragma unroll
        for (int c = 0; c < 8; ++c)
          if (c * 32 < BN) wgmma_m64n32_ss_bf16(acc[c], da, wg_desc(sa + GM_A_BYTES + c * 4096 + k * 32, 16, 1024));
      }
      wg_commit();
      wg_wait_all();
#pragma unroll
      for (int c = 0; c < 8; ++c) wg_fence_regs(acc[c]);
      __syncwarp();
      if (lane == 0) mbar_arrive(EMPTY(s));
    }
    GM_STAMP(3, 0);
    if (split_k == 1) {
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        if (c * 32 >= BN) continue;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int n = n0 + c * 32 + 8 * i;          // N % 8 == 0: a group of 8 columns is all in or all out
          if (n >= N) continue;
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const int r = row0 + 8 * rr;
            if (r < M) *reinterpret_cast<uint32_t*>(C + (size_t)r * ldc + n + 2 * t) = pack2_bf16(acc[c][4 * i + 2 * rr], acc[c][4 * i + 2 * rr + 1]);
          }
        }
      }
    }
  }
  GM_STAMP(4, 0);

  if (split_k > 1) {
    __syncthreads();   // every warpgroup is done reading the stages before they are overwritten
    if (warp < 8 && wg < n_wg) {
      // stage the fp32 partial tile over the (now idle) pipeline stages: row stride BN + 4 floats
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        if (c * 32 >= BN) continue;
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int rr = 0; rr < 2; ++rr)
            *reinterpret_cast<float2*>(reinterpret_cast<float*>(smem) + (size_t)(row0 + 8 * rr) * (BN + 4) + c * 32 + 8 * i + 2 * t) =
                make_float2(acc[c][4 * i + 2 * rr], acc[c][4 * i + 2 * rr + 1]);
      }
    }
    GM_STAMP(5, 0);
    cluster_arrive();
    cluster_wait();
    GM_STAMP(6, 0);
    // CTA y of the cluster (= the K splits of one N tile) sums rows [y * 128 / split_k, ...) over all splits
    if (split_k == 2) reduce_splits<2>(C, smem_base, BN, M, N, ldc, n0, blockIdx.y);
    else if (split_k == 4) reduce_splits<4>(C, smem_base, BN, M, N, ldc, n0, blockIdx.y);
    else reduce_splits<8>(C, smem_base, BN, M, N, ldc, n0, blockIdx.y);
    cluster_arrive();   // siblings may still be reading this CTA's partial tile
    cluster_wait();
  }
  GM_STAMP(7, 0);
}

int gemm_tc_set_timing_buffer(void* dev_ptr) {
  long long* p = reinterpret_cast<long long*>(dev_ptr);
  cudaError_t e = cudaMemcpyToSymbol(g_gemm_timing, &p, sizeof(p));
  if (e != cudaSuccess) { set_cuda_error(e, "cudaMemcpyToSymbol(g_gemm_timing)"); return LADE_ECUDA; }
  return LADE_OK;
}

// ---- host ---------------------------------------------------------------------------------------------
struct Map2Key {
  const void* ptr; int rows; int cols; int box_rows;
  bool operator==(const Map2Key& o) const { return ptr == o.ptr && rows == o.rows && cols == o.cols && box_rows == o.box_rows; }
};
struct Map2KeyHash {
  size_t operator()(const Map2Key& k) const {
    return std::hash<const void*>()(k.ptr) ^ (std::hash<int>()(k.rows) * 31) ^ (std::hash<int>()(k.cols) * 131) ^
           (std::hash<int>()(k.box_rows) * 8191);
  }
};

// [rows][cols] bf16 row-major, box = 64 cols x box_rows, SWIZZLE_128B; out-of-range rows are zero filled
static int get_tensor_map_2d(const void* ptr, int rows, int cols, int box_rows, bool streaming, CUtensorMap* out) {
  static std::mutex mu;
  static std::unordered_map<Map2Key, CUtensorMap, Map2KeyHash> cache;
  std::lock_guard<std::mutex> lock(mu);
  Map2Key key{ptr, rows, cols, box_rows};
  auto it = cache.find(key);
  if (it != cache.end()) { *out = it->second; return LADE_OK; }
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return LADE_EUNSUPPORTED;
  CUtensorMap tm;
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
  const cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   streaming ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return LADE_ECUDA;
  if (cache.size() > 8192) cache.clear();
  cache.emplace(key, tm);
  *out = tm;
  return LADE_OK;
}

static int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

static void fill_launch_config(cudaLaunchConfig_t* cfg, cudaLaunchAttribute* attr, dim3 grid, int smem, int sk, cudaStream_t stream) {
  *cfg = cudaLaunchConfig_t{};
  cfg->gridDim = grid;
  cfg->blockDim = dim3(GM_THREADS);
  cfg->dynamicSmemBytes = smem;
  cfg->stream = stream;
  attr[0].id = cudaLaunchAttributeClusterDimension;   // the K splits of one N tile form a cluster
  attr[0].val.clusterDim.x = 1;
  attr[0].val.clusterDim.y = sk;
  attr[0].val.clusterDim.z = 1;
  cfg->attrs = attr;
  cfg->numAttrs = 1;
}

static int ensure_func_attrs() {
  static unsigned long long attr_devs = 0;   // the attribute is per device (context): one bit per ordinal
  int cur_dev = 0;
  LADE_CUDA_CHECK(cudaGetDevice(&cur_dev));
  if (!((attr_devs >> (cur_dev & 63)) & 1ull)) {
    LADE_CUDA_CHECK(cudaFuncSetAttribute(gemm_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GM_SMEM_LIMIT));
    attr_devs |= 1ull << (cur_dev & 63);
  }
  return LADE_OK;
}

// CTAs of one wave for clusters of `sk` CTAs at one CTA per SM (GPC boundaries cost a few SMs per cluster shape).
static int wave_capacity(int sk) {
  static int cache[9] = {};
  if (cache[sk]) return cache[sk];
  int cap = sm_count();
  if (sk > 1) {
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute attr[1];
    fill_launch_config(&cfg, attr, dim3(64, sk, 1), GM_SMEM_LIMIT - 1024, sk, nullptr);
    int clusters = 0;
    if (cudaOccupancyMaxActiveClusters(&clusters, gemm_tc_kernel, &cfg) == cudaSuccess && clusters > 0) cap = clusters * sk;
    else { cudaGetLastError(); cap = (sm_count() / sk) * sk * 7 / 8; }
  }
  cache[sk] = cap;
  return cap;
}

// Tile width / K split so that the grid fills one wave of SMs; ties go to the wider tile (fewer re-reads of the
// activations from L2), then to the shallower split.
static void pick_config(int N, int K, int* bn_out, int* sk_out) {
  const int kb = K / GM_BK;
  int best_ctas = 0, best_bn = 256, best_sk = 1;
  for (int sk = 1; sk <= 8; sk *= 2) {
    if (kb % sk) continue;
    if (sk > 1 && kb / sk < 8) continue;
    const int cap = wave_capacity(sk);
    for (int bn = 256; bn >= 32; bn -= 32) {
      const int ctas = ((N + bn - 1) / bn) * sk;
      if (ctas > cap) continue;
      if (ctas > best_ctas || (ctas == best_ctas && bn > best_bn)) { best_ctas = ctas; best_bn = bn; best_sk = sk; }
    }
  }
  *bn_out = best_bn;
  *sk_out = best_sk;
}

int gemm_tc_launch(cudaStream_t stream, const void* a, const void* w, void* c, int M, int a_rows, int N, int K, int ldc, int bn_force,
                   int sk_force, int stages_force, int flags) {
  if (M <= 0 || M > 128 || a_rows < M || N <= 0 || K <= 0 || (K % GM_BK) || (N % 8) || (ldc % 8) || ldc < N) return LADE_EUNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(a) & 15) || (reinterpret_cast<uintptr_t>(w) & 15) || (reinterpret_cast<uintptr_t>(c) & 15))
    return LADE_EINVAL;
  int rc;
  if ((rc = ensure_func_attrs()) != LADE_OK) return rc;
  int BN, SK;
  pick_config(N, K, &BN, &SK);
  if (bn_force > 0 || sk_force > 0) {   // explicit configuration: an unspecified split defaults to 1
    if (bn_force > 0) BN = bn_force;
    SK = sk_force > 0 ? sk_force : 1;
  }
  const int kb = K / GM_BK;
  if (BN < 32 || BN > 256 || (BN % 32) || SK < 1 || SK > 8 || (SK & (SK - 1)) || (kb % SK)) return LADE_EINVAL;
  const int kbs = kb / SK;
  const int stage_bytes = GM_A_BYTES + BN * 128;
  int stages = (GM_SMEM_LIMIT - GM_BAR_BYTES - 1024) / stage_bytes;
  if (stages_force > 0 && stages_force < stages) stages = stages_force;
  if (stages > GM_MAX_STAGES) stages = GM_MAX_STAGES;
  if (stages > kbs) stages = kbs;
  if (stages < 1) return LADE_EINVAL;
  if (SK > 1 && 128 * (BN + 4) * 4 > stages * stage_bytes) return LADE_EINVAL;
  const int smem = stages * stage_bytes + GM_BAR_BYTES + 1024;   // + slack to align the base to 1024 bytes

  CUtensorMap tmA, tmW;
  if ((rc = get_tensor_map_2d(a, a_rows, K, 128, false, &tmA)) != LADE_OK) return rc;
  if ((rc = get_tensor_map_2d(w, N, K, BN, true, &tmW)) != LADE_OK) return rc;
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  fill_launch_config(&cfg, attr, dim3((N + BN - 1) / BN, SK, 1), smem, SK, stream);
  static int launch_counter = 0;
  const int prefill = (flags & 1) ? 0 : 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, gemm_tc_kernel, tmA, tmW, (__nv_bfloat16*)c, M, N, ldc, kbs, BN, stages, SK, prefill,
                                     launch_counter++);
  if (e != cudaSuccess) { set_cuda_error(e, "cudaLaunchKernelEx(gemm_tc_kernel)"); return LADE_ECUDA; }
  return LADE_OK;
}

}  // namespace lade

extern "C" int lade_debug_gemm_timing(void* dev_buffer) { return lade::gemm_tc_set_timing_buffer(dev_buffer); }

extern "C" int lade_gemm_bf16(void* stream, const void* a, const void* w, void* c, int32_t m, int32_t a_rows, int32_t n, int32_t k,
                              int32_t ldc, int32_t tile_n, int32_t split_k) {
  return lade::gemm_tc_launch(reinterpret_cast<cudaStream_t>(stream), a, w, c, m, a_rows, n, k, ldc, tile_n & 0xffff, split_k, (tile_n >> 16) & 15,
                              (tile_n >> 20) & 15);
}
