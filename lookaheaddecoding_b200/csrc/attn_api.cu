// C-ABI dispatch of the lookahead attention kernels.
#include "common.cuh"

namespace lade {
int attn_fwd_mma_launch(cudaStream_t stream, const void* q, const void* k_cache, const void* v_cache, void* out,
                        const uint32_t* rowmask, int mask_words, const int32_t* meta, void* scratch, int q_pad, int n_heads,
                        int n_kv_heads, int head_dim, int kv_capacity, int n_splits, int is_f16);
int attn_fwd_tc_launch(cudaStream_t stream, const void* q, const void* k_cache, const void* v_cache, void* out,
                       const uint32_t* rowmask, int mask_words, const int32_t* meta, void* scratch, int q_pad, int n_heads,
                       int n_kv_heads, int head_dim, int kv_capacity, int kv_bound, int n_splits, int is_f16);
int attn_fwd_tc_exact_launch(cudaStream_t stream, const void* q, const void* k_cache, const void* v_cache, void* out,
                             const uint32_t* rowmask, int mask_words, const int32_t* meta, void* scratch, int q_pad, int n_heads,
                             int n_kv_heads, int head_dim, int kv_capacity, int kv_bound, int n_splits, int is_f16);
int attn_tc_set_timing_buffer(void* dev_ptr);
int attn_tc_set_pdl(int v);
}  // namespace lade

extern "C" {

int lade_debug_attn_timing(void* dev_buffer) { return lade::attn_tc_set_timing_buffer(dev_buffer); }

int lade_debug_attn_pdl(int32_t enable) { return lade::attn_tc_set_pdl(enable); }


int64_t lade_attn_scratch_bytes(int32_t q_pad, int32_t n_heads, int32_t head_dim, int32_t n_splits) {
  if (q_pad < 1 || n_heads < 1 || head_dim < 1 || n_splits < 1) return LADE_EINVAL;
  const int64_t rows_pad = (int64_t)((q_pad + 127) / 128) * 128;
  return 16384 * 4 + (int64_t)n_splits * n_heads * rows_pad * (head_dim + 2) * 4;
}

int lade_attn_fwd(void* stream, const void* q, const void* k_cache, const void* v_cache, void* out,
                  const uint32_t* rowmask, int32_t mask_words, const int32_t* meta, void* scratch, int32_t q_pad,
                  int32_t n_heads, int32_t n_kv_heads, int32_t head_dim, int32_t kv_capacity,
                  int32_t kv_bound, int32_t n_splits, int32_t impl) {
  if (!q || !k_cache || !v_cache || !out || !meta || !scratch) return LADE_EINVAL;
  if (rowmask && mask_words * 32 < q_pad) return LADE_EINVAL;   // rowmask may be NULL for prefill-only use
  if (q_pad < 1 || n_heads < 1 || n_kv_heads < 1 || n_heads % n_kv_heads != 0 || n_splits < 1 || kv_capacity < 1)
    return LADE_EINVAL;
  // impl 0 = the library's choice: the Hopper-native wgmma/TMA kernel for head_dim 128, the mma.sync kernel for the
  // other instantiated head dimension (64); impl 2 / 1 force one of them; impl 3 = the wgmma kernel's reference-order
  // variant (probabilities normalised before they are rounded, like modeling_llama.py:530-541; kv_bound must bound
  // kv_len + q_len and fit 384 * n_splits)
  if (impl == 3)
    return lade::attn_fwd_tc_exact_launch((cudaStream_t)stream, q, k_cache, v_cache, out, rowmask, mask_words, meta, scratch,
                                          q_pad, n_heads, n_kv_heads, head_dim, kv_capacity, kv_bound, n_splits, 0);
  if ((impl == 0 && head_dim == 128) || impl == 2)
    return lade::attn_fwd_tc_launch((cudaStream_t)stream, q, k_cache, v_cache, out, rowmask, mask_words, meta, scratch, q_pad,
                                    n_heads, n_kv_heads, head_dim, kv_capacity, kv_bound, n_splits, 0);
  return lade::attn_fwd_mma_launch((cudaStream_t)stream, q, k_cache, v_cache, out, rowmask, mask_words, meta, scratch, q_pad,
                                   n_heads, n_kv_heads, head_dim, kv_capacity, n_splits, 0);
}

/* fp16 models: the same attention with every rounding point in fp16 (the reference runs the module in the model dtype).
 * Same choice of kernel as the bf16 entry point: wgmma/TMA for head_dim 128 (impl 0 or 2), mma.sync otherwise. */
int lade_attn_fwd_f16(void* stream, const void* q, const void* k_cache, const void* v_cache, void* out,
                      const uint32_t* rowmask, int32_t mask_words, const int32_t* meta, void* scratch, int32_t q_pad,
                      int32_t n_heads, int32_t n_kv_heads, int32_t head_dim, int32_t kv_capacity,
                      int32_t kv_bound, int32_t n_splits, int32_t impl) {
  if (!q || !k_cache || !v_cache || !out || !meta || !scratch) return LADE_EINVAL;
  if (rowmask && mask_words * 32 < q_pad) return LADE_EINVAL;
  if (q_pad < 1 || n_heads < 1 || n_kv_heads < 1 || n_heads % n_kv_heads != 0 || n_splits < 1 || kv_capacity < 1)
    return LADE_EINVAL;
  if (impl == 3)
    return lade::attn_fwd_tc_exact_launch((cudaStream_t)stream, q, k_cache, v_cache, out, rowmask, mask_words, meta, scratch,
                                          q_pad, n_heads, n_kv_heads, head_dim, kv_capacity, kv_bound, n_splits, 1);
  if ((impl == 0 && head_dim == 128) || impl == 2)
    return lade::attn_fwd_tc_launch((cudaStream_t)stream, q, k_cache, v_cache, out, rowmask, mask_words, meta, scratch, q_pad,
                                    n_heads, n_kv_heads, head_dim, kv_capacity, kv_bound, n_splits, 1);
  return lade::attn_fwd_mma_launch((cudaStream_t)stream, q, k_cache, v_cache, out, rowmask, mask_words, meta, scratch, q_pad,
                                   n_heads, n_kv_heads, head_dim, kv_capacity, n_splits, 1);
}

}  // extern "C"
