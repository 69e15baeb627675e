// Shared helpers for the lade sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include "../../include/lade_sm100.h"

namespace lade {

void set_cuda_error(cudaError_t e, const char* where);
void set_error_string(const char* msg);      // shown by lade_last_cuda_error() (also used for NCCL failures)

#define LADE_CUDA_CHECK(expr)                                   \
  do {                                                          \
    cudaError_t _e = (expr);                                    \
    if (_e != cudaSuccess) {                                    \
      ::lade::set_cuda_error(_e, #expr);                        \
      return LADE_ECUDA;                                        \
    }                                                           \
  } while (0)

#define LADE_LAUNCH_CHECK(name)                                 \
  do {                                                          \
    cudaError_t _e = cudaGetLastError();                        \
    if (_e != cudaSuccess) {                                    \
      ::lade::set_cuda_error(_e, name);                         \
      return LADE_ECUDA;                                        \
    }                                                           \
  } while (0)

__host__ __device__ inline int rowdesc_make(int cls, int blk, int idx) {
  return (int)(((unsigned)cls << 30) | ((unsigned)blk << 15) | (unsigned)idx);
}
__host__ __device__ inline int rowdesc_cls(int rd) { return (int)((unsigned)rd >> 30); }
__host__ __device__ inline int rowdesc_blk(int rd) { return (int)(((unsigned)rd >> 15) & 0x7fffu); }
__host__ __device__ inline int rowdesc_idx(int rd) { return (int)((unsigned)rd & 0x7fffu); }

// Lookahead mask predicate over step-local (row r, column c); SURVEY.md App. B ==
// j_make_causal_mask_multilevel (lade/models/modeling_llama.py:115-207).  Cache columns are
// visible to every row and never reach this function.
__device__ __forceinline__ bool row_sees(int rd_r, int r, int rd_c, int c, int level_offset) {
  const int tr = rowdesc_cls(rd_r);
  const int tc = rowdesc_cls(rd_c);
  if (tr == LADE_ROW_PREFIX) return tc == LADE_ROW_PREFIX && c <= r;        // :124-130, :189-192
  if (tr == LADE_ROW_WINDOW) {
    if (tc == LADE_ROW_PREFIX) return true;                                 // :195
    if (tc != LADE_ROW_WINDOW) return false;
    const int bc = rowdesc_blk(rd_c), ic = rowdesc_idx(rd_c);
    const int br = rowdesc_blk(rd_r), ir = rowdesc_idx(rd_r);
    return bc == 0 ? (ic <= ir) : (bc <= br && ic == ir);                   // :201-203
  }
  if (tr == LADE_ROW_GUESS) {
    if (c <= level_offset) return true;                                     // :184
    return tc == LADE_ROW_GUESS && rowdesc_blk(rd_c) == rowdesc_blk(rd_r) &&
           rowdesc_idx(rd_c) <= rowdesc_idx(rd_r);                          // :141-181
  }
  return c == r;  // PAD rows only see themselves
}

// 32 visibility bits of one query row for cache/step columns [col, col+32).
//   rowmask row: bit c of word c/32 = row sees step column c (c < q_len), built by lade_step_layout from
//   row_sees(); cache columns (col < kv_len) are visible to every row, columns >= kv_len + q_len to none.
//   Prefill steps carry no rowmask: plain causal (modeling_llama.py:124-130).
__device__ __forceinline__ uint32_t visible_bits32(const uint32_t* __restrict__ mrow, int mask_words, int col, int kv_len,
                                                   int q_len, int is_prefill, int row) {
  const int cs = col - kv_len;                       // first step column of the chunk (may be negative)
  if (cs + 32 <= 0) return 0xffffffffu;
  uint32_t step_bits;                                // visibility of step columns max(cs,0) .. cs+31, bit i <-> cs+i
  if (is_prefill) {
    const int n = (row < q_len ? row : -1) - cs + 1; // columns c <= row are visible
    step_bits = n <= 0 ? 0u : (n >= 32 ? 0xffffffffu : ((1u << n) - 1u));
    if (row >= q_len) step_bits = 0u;
    const int nq = q_len - cs;                       // clip at q_len
    if (nq < 32) step_bits &= nq <= 0 ? 0u : ((1u << nq) - 1u);
    if (cs < 0) step_bits |= (1u << (-cs)) - 1u;
    return step_bits;
  }
  if (!mrow) return cs < 0 ? ((1u << (-cs)) - 1u) : 0u;
  if (cs < 0) {
    const int k = -cs;
    return ((1u << k) - 1u) | (mrow[0] << k);
  }
  const int w = cs >> 5, sh = cs & 31;
  const uint32_t lo = w < mask_words ? mrow[w] : 0u;
  const uint32_t hi = (w + 1) < mask_words ? mrow[w + 1] : 0u;
  return __funnelshift_r(lo, hi, sh);
}

__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// Element type of a model (bf16 or fp16): conversions with the rounding the reference's tensors get (round to nearest
// even into the model dtype after every op, lade/models/modeling_llama.py runs in `torch_dtype`).
template <typename T> struct Elem;
template <> struct Elem<__nv_bfloat16> {
  static __device__ __forceinline__ float to_f(__nv_bfloat16 x) { return __bfloat162float(x); }
  static __device__ __forceinline__ __nv_bfloat16 from_f(float x) { return __float2bfloat16_rn(x); }
  static __device__ __forceinline__ unsigned pack2(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<unsigned*>(&v);
  }
  static __device__ __forceinline__ unsigned key16(__nv_bfloat16 x) { return __bfloat16_as_ushort(x); }
};
template <> struct Elem<__half> {
  static __device__ __forceinline__ float to_f(__half x) { return __half2float(x); }
  static __device__ __forceinline__ __half from_f(float x) { return __float2half_rn(x); }
  static __device__ __forceinline__ unsigned pack2(float lo, float hi) {
    __half2 v = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<unsigned*>(&v);
  }
  static __device__ __forceinline__ unsigned key16(__half x) { return __half_as_ushort(x); }
};
template <typename T> __device__ __forceinline__ float round_to(float x) { return Elem<T>::to_f(Elem<T>::from_f(x)); }

}  // namespace lade
