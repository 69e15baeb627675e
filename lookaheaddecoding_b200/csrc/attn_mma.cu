// Lookahead attention, legacy tensor-core path (mma.sync m16n8k16, cp.async staging).
//
// This is the robust first implementation (impl=1): split-KV flash attention over the persistent
// KV cache with the lookahead mask evaluated in registers.  The wgmma/TMA implementation
// (attn_tc.cu, impl=2) is validated against it.  Replaces the attention core of
// LlamaAttention.forward (lade/models/modeling_llama.py:520-541) + the dense additive mask of
// j_make_causal_mask_multilevel (:115-207).
//
// Head dimensions 128 (Llama-2/3, CodeLlama) and 64 (TinyLlama-style) are instantiated; the wgmma path is built for
// 128 only, so 64 always runs here.
//
// Rounding points follow the reference: scores = bf16(QK^T) ; bf16(scores * (1/sqrt(D))) (torch's
// CUDA division-by-scalar multiplies by the fp32 reciprocal) ; fp32 softmax ; bf16 probabilities ;
// fp32-accumulated PV ; bf16 output.
#include "common.cuh"

namespace lade {

constexpr int ATT_BM = 128;
constexpr int ATT_BN = 64;
constexpr int ATT_STAGES = 3;
constexpr int ATT_THREADS = 256;
constexpr int ATT_RD_SMEM = 1024;
constexpr int ATTN_MAX_COUNTERS = 16384;

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, int src_bytes) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ void ldmatrix_x4(unsigned& r0, unsigned& r1, unsigned& r2, unsigned& r3, const void* p) {
  const unsigned a = (unsigned)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(a));
}
__device__ __forceinline__ void ldmatrix_x4_trans(unsigned& r0, unsigned& r1, unsigned& r2, unsigned& r3, const void* p) {
  const unsigned a = (unsigned)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(a));
}
template <typename T>
__device__ __forceinline__ void mma_16816(float (&c)[4], const unsigned (&a)[4], unsigned b0, unsigned b1);
template <>
__device__ __forceinline__ void mma_16816<__nv_bfloat16>(float (&c)[4], const unsigned (&a)[4], unsigned b0, unsigned b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <>
__device__ __forceinline__ void mma_16816<__half>(float (&c)[4], const unsigned (&a)[4], unsigned b0, unsigned b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// swizzled element offset inside a [BN][ATT_D] bf16 tile: 16-byte chunk index XOR (row & 7)
template <int ATT_D>
__device__ __forceinline__ int swz(int row, int chunk) { return row * ATT_D + ((chunk ^ (row & 7)) << 3); }

template <int ATT_D, typename T>
__device__ __forceinline__ void load_tile_async(T* sK, T* sV, const T* gK, const T* gV, int row0, int T_rows, int kv_capacity) {
  // 64 rows x (ATT_D / 8) 16-byte chunks per tensor; 256 threads -> 4 (D = 128) or 2 (D = 64) chunks each per tensor
  constexpr int CPR = ATT_D / 8;
#pragma unroll
  for (int i = 0; i < (ATT_BN * CPR) / ATT_THREADS; ++i) {
    const int c = threadIdx.x + i * ATT_THREADS;
    const int row = c / CPR, chunk = c % CPR;
    const int grow = row0 + row;
    const int ok = (grow < T_rows) ? 16 : 0;
    const int crow = grow < kv_capacity ? grow : kv_capacity - 1;
    cp_async16(sK + swz<ATT_D>(row, chunk), gK + (long long)crow * ATT_D + chunk * 8, ok);
    cp_async16(sV + swz<ATT_D>(row, chunk), gV + (long long)crow * ATT_D + chunk * 8, ok);
  }
}

template <int ATT_D, typename ET>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_mma_kernel(const ET* __restrict__ q, const ET* __restrict__ k_cache,
                    const ET* __restrict__ v_cache, ET* __restrict__ out,
                    const uint32_t* __restrict__ rowmask, int mask_words, const int* __restrict__ meta,
                    float* __restrict__ part_o,
                    float* __restrict__ part_ml, int* __restrict__ counters, int q_pad, int n_heads,
                    int n_kv_heads, int kv_capacity, int n_splits, float inv_sqrt_d) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  ET* sK = reinterpret_cast<ET*>(smem_raw);
  ET* sV = sK + ATT_STAGES * ATT_BN * ATT_D;
  __shared__ int s_last;

  const int split = blockIdx.x, h = blockIdx.y, mt = blockIdx.z;
  const int q_tiles = gridDim.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q_len = meta[LADE_M_Q_LEN];
  const int kv_len = meta[LADE_M_KV_LEN];
  const int is_prefill = meta[LADE_M_IS_PREFILL];
  const int T = kv_len + q_len;
  int Tm = T;
  if (is_prefill) {  // causal: rows of this q tile see nothing past their own column
    const int lim = kv_len + min(q_len, (mt + 1) * ATT_BM);
    Tm = min(T, lim);
  }
  const int n_tiles = (Tm + ATT_BN - 1) / ATT_BN;
  const int tps = (n_tiles + n_splits - 1) / n_splits;
  const int n_active = (n_tiles + tps - 1) / tps;
  if (split >= n_active) return;
  const int tile_lo = split * tps;
  const int tile_hi = min(n_tiles, tile_lo + tps);
  const int my_tiles = tile_hi - tile_lo;

  const int hk = h / (n_heads / n_kv_heads);
  const ET* gK = k_cache + (long long)hk * kv_capacity * ATT_D;
  const ET* gV = v_cache + (long long)hk * kv_capacity * ATT_D;

  // prologue: prefetch up to STAGES-1 tiles
#pragma unroll
  for (int s = 0; s < ATT_STAGES - 1; ++s) {
    if (s < my_tiles)
      load_tile_async<ATT_D, ET>(sK + s * ATT_BN * ATT_D, sV + s * ATT_BN * ATT_D, gK, gV, (tile_lo + s) * ATT_BN, T, kv_capacity);
    cp_async_commit();
  }

  // Q fragments (A operand), 16 rows per warp
  const int row_a = mt * ATT_BM + warp * 16 + (lane >> 2);  // step-local row of c0/c1
  const int row_b = row_a + 8;
  constexpr int KK = ATT_D / 16;       // k16 steps of QK^T
  constexpr int ND = ATT_D / 8;        // 8-wide n-tiles of the output
  unsigned qf[KK][4];
  {
    const ET* qh = q + (long long)h * q_pad * ATT_D;
#pragma unroll
    for (int kk = 0; kk < KK; ++kk) {
      const int col = kk * 16 + (lane & 3) * 2;
      qf[kk][0] = row_a < q_pad ? *reinterpret_cast<const unsigned*>(qh + (long long)row_a * ATT_D + col) : 0u;
      qf[kk][1] = row_b < q_pad ? *reinterpret_cast<const unsigned*>(qh + (long long)row_b * ATT_D + col) : 0u;
      qf[kk][2] = row_a < q_pad ? *reinterpret_cast<const unsigned*>(qh + (long long)row_a * ATT_D + col + 8) : 0u;
      qf[kk][3] = row_b < q_pad ? *reinterpret_cast<const unsigned*>(qh + (long long)row_b * ATT_D + col + 8) : 0u;
    }
  }
  const bool have_mask = (!is_prefill) && rowmask != nullptr;
  const uint32_t* mrow_a = (have_mask && row_a < q_pad) ? rowmask + (long long)row_a * mask_words : nullptr;
  const uint32_t* mrow_b = (have_mask && row_b < q_pad) ? rowmask + (long long)row_b * mask_words : nullptr;

  float o_acc[ND][4];
#pragma unroll
  for (int i = 0; i < ND; ++i) { o_acc[i][0] = o_acc[i][1] = o_acc[i][2] = o_acc[i][3] = 0.f; }
  float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f;
  const float LOG2E = 1.4426950408889634f;

  for (int it = 0; it < my_tiles; ++it) {
    // prefetch tile it + STAGES-1
    {
      const int nt = it + ATT_STAGES - 1;
      if (nt < my_tiles) {
        const int st = nt % ATT_STAGES;
        load_tile_async<ATT_D, ET>(sK + st * ATT_BN * ATT_D, sV + st * ATT_BN * ATT_D, gK, gV, (tile_lo + nt) * ATT_BN, T, kv_capacity);
      }
      cp_async_commit();
    }
    cp_async_wait<ATT_STAGES - 1>();
    __syncthreads();
    const int st = it % ATT_STAGES;
    const ET* tK = sK + st * ATT_BN * ATT_D;
    const ET* tV = sV + st * ATT_BN * ATT_D;
    const int col0 = (tile_lo + it) * ATT_BN;

    // ---- S = Q K^T
    float s_acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s_acc[i][0] = s_acc[i][1] = s_acc[i][2] = s_acc[i][3] = 0.f; }
#pragma unroll
    for (int kk = 0; kk < KK; ++kk) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {  // pairs of n-tiles
        unsigned b0, b1, b2, b3;
        const int m = lane >> 3, r = lane & 7;
        const int row = np * 16 + (m >> 1) * 8 + r;
        const int chunk = kk * 2 + (m & 1);
        ldmatrix_x4(b0, b1, b2, b3, tK + swz<ATT_D>(row, chunk));
        mma_16816<ET>(s_acc[np * 2], qf[kk], b0, b1);
        mma_16816<ET>(s_acc[np * 2 + 1], qf[kk], b2, b3);
      }
    }

    // ---- reference rounding + mask: 64 visibility bits per row for this tile, tested in registers
    const bool need_mask = (col0 + ATT_BN > kv_len);
    unsigned long long va = ~0ull, vb = ~0ull;
    if (need_mask) {
      va = (unsigned long long)visible_bits32(mrow_a, mask_words, col0, kv_len, q_len, is_prefill, row_a) |
           ((unsigned long long)visible_bits32(mrow_a, mask_words, col0 + 32, kv_len, q_len, is_prefill, row_a) << 32);
      vb = (unsigned long long)visible_bits32(mrow_b, mask_words, col0, kv_len, q_len, is_prefill, row_b) |
           ((unsigned long long)visible_bits32(mrow_b, mask_words, col0 + 32, kv_len, q_len, is_prefill, row_b) << 32);
    }
    va >>= (lane & 3) * 2;   // this thread's two columns of every 8-wide n-tile
    vb >>= (lane & 3) * 2;
    float mx_a = -INFINITY, mx_b = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float s = round_to<ET>(round_to<ET>(s_acc[nt][e]) * inv_sqrt_d);
        const unsigned long long vv = (e < 2) ? va : vb;
        if (!((vv >> (nt * 8 + (e & 1))) & 1ull)) s = -INFINITY;
        s_acc[nt][e] = s;
        if (e < 2) mx_a = fmaxf(mx_a, s); else mx_b = fmaxf(mx_b, s);
      }
    }
    mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 1));
    mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 2));
    mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 1));
    mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 2));
    const float mn_a = fmaxf(m_a, mx_a), mn_b = fmaxf(m_b, mx_b);
    const float sc_a = (mn_a == -INFINITY) ? 1.f : exp2f((m_a - mn_a) * LOG2E);
    const float sc_b = (mn_b == -INFINITY) ? 1.f : exp2f((m_b - mn_b) * LOG2E);
    const float off_a = (mn_a == -INFINITY) ? 0.f : mn_a * LOG2E;
    const float off_b = (mn_b == -INFINITY) ? 0.f : mn_b * LOG2E;
    m_a = mn_a; m_b = mn_b;
    float ps_a = 0.f, ps_b = 0.f;
    unsigned pf[4][4];  // A fragments of P for the 4 k16 steps over this tile's 64 kv rows
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float p0 = exp2f(s_acc[nt][0] * LOG2E - off_a);
      const float p1 = exp2f(s_acc[nt][1] * LOG2E - off_a);
      const float p2 = exp2f(s_acc[nt][2] * LOG2E - off_b);
      const float p3 = exp2f(s_acc[nt][3] * LOG2E - off_b);
      ps_a += p0 + p1;
      ps_b += p2 + p3;
      const int ks = nt >> 1;
      if ((nt & 1) == 0) { pf[ks][0] = Elem<ET>::pack2(p0, p1); pf[ks][1] = Elem<ET>::pack2(p2, p3); }
      else               { pf[ks][2] = Elem<ET>::pack2(p0, p1); pf[ks][3] = Elem<ET>::pack2(p2, p3); }
    }
    l_a = l_a * sc_a + ps_a;
    l_b = l_b * sc_b + ps_b;
#pragma unroll
    for (int i = 0; i < ND; ++i) {
      o_acc[i][0] *= sc_a; o_acc[i][1] *= sc_a; o_acc[i][2] *= sc_b; o_acc[i][3] *= sc_b;
    }

    // ---- O += P V
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
      for (int nd = 0; nd < ND / 2; ++nd) {  // pairs of d n-tiles
        unsigned b0, b1, b2, b3;
        const int m = lane >> 3, r = lane & 7;
        const int row = ks * 16 + (m & 1) * 8 + r;
        const int chunk = nd * 2 + (m >> 1);
        ldmatrix_x4_trans(b0, b1, b2, b3, tV + swz<ATT_D>(row, chunk));
        mma_16816<ET>(o_acc[nd * 2], pf[ks], b0, b1);
        mma_16816<ET>(o_acc[nd * 2 + 1], pf[ks], b2, b3);
      }
    }
    __syncthreads();  // stage may be overwritten by the next prefetch
  }
  cp_async_wait<0>();

  // row sums across the quad
  l_a += __shfl_xor_sync(0xffffffffu, l_a, 1);
  l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
  l_b += __shfl_xor_sync(0xffffffffu, l_b, 1);
  l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);

  const int HD = n_heads * ATT_D;
  if (n_active == 1) {
    const float inv_a = l_a > 0.f ? 1.f / l_a : 0.f;
    const float inv_b = l_b > 0.f ? 1.f / l_b : 0.f;
#pragma unroll
    for (int nt = 0; nt < ND; ++nt) {
      const int col = nt * 8 + (lane & 3) * 2;
      if (row_a < q_pad)
        *reinterpret_cast<unsigned*>(out + (long long)row_a * HD + h * ATT_D + col) = Elem<ET>::pack2(o_acc[nt][0] * inv_a, o_acc[nt][1] * inv_a);
      if (row_b < q_pad)
        *reinterpret_cast<unsigned*>(out + (long long)row_b * HD + h * ATT_D + col) = Elem<ET>::pack2(o_acc[nt][2] * inv_b, o_acc[nt][3] * inv_b);
    }
    return;
  }

  // ---- split-KV partials (unnormalised O, running max, running sum), combined by the last CTA
  const int rows_pad = q_tiles * ATT_BM;
  {
    float* po = part_o + (((long long)split * n_heads + h) * rows_pad) * ATT_D;
    float* pml = part_ml + (((long long)split * n_heads + h) * rows_pad) * 2;
#pragma unroll
    for (int nt = 0; nt < ND; ++nt) {
      const int col = nt * 8 + (lane & 3) * 2;
      *reinterpret_cast<float2*>(po + (long long)row_a * ATT_D + col) = make_float2(o_acc[nt][0], o_acc[nt][1]);
      *reinterpret_cast<float2*>(po + (long long)row_b * ATT_D + col) = make_float2(o_acc[nt][2], o_acc[nt][3]);
    }
    if ((lane & 3) == 0) {
      *reinterpret_cast<float2*>(pml + (long long)row_a * 2) = make_float2(m_a, l_a);
      *reinterpret_cast<float2*>(pml + (long long)row_b * 2) = make_float2(m_b, l_b);
    }
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int prev = atomicAdd(&counters[h * q_tiles + mt], 1);
    s_last = (prev == n_active - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // combine: thread -> (row, 4 columns)
  for (int idx = threadIdx.x; idx < ATT_BM * (ATT_D / 4); idx += ATT_THREADS) {
    const int rl = idx / (ATT_D / 4), c4 = idx % (ATT_D / 4);
    const int row = mt * ATT_BM + rl;
    if (row >= q_pad) continue;
    float mmax = -INFINITY;
    for (int s = 0; s < n_active; ++s) {
      const float ms = __ldcg(part_ml + ((((long long)s * n_heads + h) * rows_pad) + row) * 2);
      mmax = fmaxf(mmax, ms);
    }
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    float lsum = 0.f;
    for (int s = 0; s < n_active; ++s) {
      const float2 ml = __ldcg(reinterpret_cast<const float2*>(part_ml + ((((long long)s * n_heads + h) * rows_pad) + row) * 2));
      const float wgt = (ml.x == -INFINITY) ? 0.f : exp2f((ml.x - mmax) * LOG2E);
      const float4 v = __ldcg(reinterpret_cast<const float4*>(part_o + ((((long long)s * n_heads + h) * rows_pad) + row) * ATT_D + c4 * 4));
      acc.x += v.x * wgt; acc.y += v.y * wgt; acc.z += v.z * wgt; acc.w += v.w * wgt;
      lsum += ml.y * wgt;
    }
    const float inv = lsum > 0.f ? 1.f / lsum : 0.f;
    uint2 pk;
    pk.x = Elem<ET>::pack2(acc.x * inv, acc.y * inv);
    pk.y = Elem<ET>::pack2(acc.z * inv, acc.w * inv);
    *reinterpret_cast<uint2*>(out + (long long)row * HD + h * ATT_D + c4 * 4) = pk;
  }
  if (threadIdx.x == 0) counters[h * q_tiles + mt] = 0;
}

template <int ATT_D, typename ET>
static int attn_fwd_mma_launch_d(cudaStream_t stream, const void* q, const void* k_cache, const void* v_cache, void* out,
                                 const uint32_t* rowmask, int mask_words, const int32_t* meta, void* scratch, int q_pad,
                                 int n_heads, int n_kv_heads, int kv_capacity, int n_splits) {
  const int q_tiles = (q_pad + ATT_BM - 1) / ATT_BM;
  const size_t smem = (size_t)2 * ATT_STAGES * ATT_BN * ATT_D * sizeof(ET);
  static unsigned long long attr_devs = 0;   // the attribute is per device (context): one bit per ordinal
  int cur_dev = 0;
  LADE_CUDA_CHECK(cudaGetDevice(&cur_dev));
  if (!((attr_devs >> (cur_dev & 63)) & 1ull)) {
    LADE_CUDA_CHECK(cudaFuncSetAttribute(attn_fwd_mma_kernel<ATT_D, ET>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_devs |= 1ull << (cur_dev & 63);
  }
  const long long rows_pad = (long long)q_tiles * ATT_BM;
  if ((long long)n_heads * q_tiles > ATTN_MAX_COUNTERS) return LADE_EUNSUPPORTED;
  // scratch = [counters (fixed region, zero at rest)] [part_ml] [part_o]
  int* counters = reinterpret_cast<int*>(scratch);
  float* part_ml = reinterpret_cast<float*>(counters + ATTN_MAX_COUNTERS);
  float* part_o = part_ml + (long long)n_splits * n_heads * rows_pad * 2;
  dim3 grid(n_splits, n_heads, q_tiles);
  attn_fwd_mma_kernel<ATT_D, ET><<<grid, ATT_THREADS, smem, stream>>>(
      (const ET*)q, (const ET*)k_cache, (const ET*)v_cache, (ET*)out,
      rowmask, mask_words, meta, part_o, part_ml, counters, q_pad, n_heads, n_kv_heads, kv_capacity, n_splits,
      1.0f / sqrtf((float)ATT_D));
  LADE_LAUNCH_CHECK("attn_fwd_mma_kernel");
  return LADE_OK;
}

int attn_fwd_mma_launch(cudaStream_t stream, const void* q, const void* k_cache, const void* v_cache, void* out,
                        const uint32_t* rowmask, int mask_words, const int32_t* meta, void* scratch, int q_pad, int n_heads,
                        int n_kv_heads, int head_dim, int kv_capacity, int n_splits, int is_f16) {
#define LADE_MMA_DISPATCH(DD, TT)                                                                                        \
  return attn_fwd_mma_launch_d<DD, TT>(stream, q, k_cache, v_cache, out, rowmask, mask_words, meta, scratch, q_pad, n_heads, \
                                       n_kv_heads, kv_capacity, n_splits)
  if (head_dim == 128) { if (is_f16) LADE_MMA_DISPATCH(128, __half); else LADE_MMA_DISPATCH(128, __nv_bfloat16); }
  if (head_dim == 64) { if (is_f16) LADE_MMA_DISPATCH(64, __half); else LADE_MMA_DISPATCH(64, __nv_bfloat16); }
#undef LADE_MMA_DISPATCH
  return LADE_EUNSUPPORTED;
}

}  // namespace lade
