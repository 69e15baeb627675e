// Per-token logits capture: after a step's commit, copy the lm-head row each emitted token was decided from into the
// caller's [generated token][ld_out] buffer, inside the step's CUDA graph.  This is what generate() returns as HF's
// `logits` / `scores` (return_dict_in_generate), which the reference refuses (lade/decoding.py:411, :967).
//
// Which slot decided emitted token j of a step (lm slot layout of lade_step_layout; guess n-gram e, token u is slot
// 1 + WCAP + e*GS + u):
//   j = 0            slot 0 on every path (prefill, window fill, steady step);
//   greedy, j >= 1   slot (max_hit_idx, j-1): accept_update emits hits[j] = argmax of that slot (state.cu,
//                    local_decision);
//   sampling, j >= 1 slot (e_{j-1}, j-1), e_i = min{e : guess[e][0..i] == hits[0..i]}: the chain of
//                    sample_verify_chain moves to the row of the candidate accepted at position i, and that is the
//                    first alive candidate carrying hits[i] (an earlier one carrying it would have been tried first,
//                    and its rejection puts the token in the zero set, so nothing could accept it afterwards).
// The guess tokens are read from the step's own rows (ids[lm_rows[slot]]), never from the ctx state, which the commit
// has already advanced.
#include "state.cuh"

#include <climits>

namespace lade {

constexpr int CAP_THREADS = 256;
constexpr int CAP_COLS = CAP_THREADS * 8;         // columns per CTA: one 16-byte vector per thread

// grid: (ceil(vocab / CAP_COLS), N-1); blockIdx.y = emitted token j of the step.
template <typename T>
__global__ void __launch_bounds__(CAP_THREADS)
capture_rows_kernel(const int* __restrict__ st, Dims d, const T* __restrict__ logits, int ld, int vocab,
                    const int* __restrict__ ids, const int* __restrict__ lm_rows, const int* __restrict__ meta,
                    const int* __restrict__ res, int sampling, T* __restrict__ out, int ld_out, int out_rows) {
  __shared__ int s_e;
  const int j = blockIdx.y;
  const int t = threadIdx.x;
  if (meta[LADE_M_DONE]) return;                  // step on a finished state (the pipelined loop's surplus step)
  const int n_emit = res[LADE_R_N_EMIT];
  if (j >= n_emit) return;
  const int row = res[LADE_R_N_OUT] - n_emit - st[S_N_PROMPT] + j;   // generated-token index of this token
  if (row < 0 || row >= out_rows) return;
  const int GS = d.GS, g_slot0 = 1 + d.WCAP;
  int slot = 0;
  if (j > 0 && !sampling) {
    slot = g_slot0 + res[LADE_R_MAX_HIT_IDX] * GS + j - 1;
  } else if (j > 0) {
    const int n_ng = meta[LADE_M_N_GUESS_TOK] / GS;
    if (t == 0) s_e = INT_MAX;
    __syncthreads();
    for (int e = t; e < n_ng; e += blockDim.x) {
      bool match = true;
      for (int u = 0; u < j && match; ++u) match = ids[lm_rows[g_slot0 + e * GS + u]] == res[LADE_R_HITS + u];
      if (match) atomicMin(&s_e, e);
    }
    __syncthreads();
    if (s_e == INT_MAX) return;                   // no candidate carries the hits: nothing was decided from a guess row
    slot = g_slot0 + s_e * GS + j - 1;
  }
  if (slot >= d.lm_cap) return;
  const T* src = logits + (long long)slot * ld;
  T* dst = out + (long long)row * ld_out;
  const int c = blockIdx.x * CAP_COLS + t * 8;
  if (c >= vocab) return;
  const bool vec = c + 8 <= vocab && ((reinterpret_cast<uintptr_t>(src + c) | reinterpret_cast<uintptr_t>(dst + c)) & 15) == 0;
  if (vec) {
    *reinterpret_cast<uint4*>(dst + c) = *reinterpret_cast<const uint4*>(src + c);
  } else {
    for (int k = c; k < min(c + 8, vocab); ++k) dst[k] = src[k];
  }
}

template <typename T>
static int launch_capture_rows(LadeCtx* ctx, void* stream, const void* logits, int32_t ld, int32_t vocab,
                               const int32_t* ids, const int32_t* lm_rows, const int32_t* meta, const int32_t* result,
                               int32_t sampling, void* out, int32_t ld_out, int32_t out_rows) {
  if (!ctx || !logits || !ids || !lm_rows || !meta || !result || !out) return LADE_EINVAL;
  if (vocab < 1 || ld < vocab || ld_out < vocab || out_rows < 1 || (sampling != 0 && sampling != 1)) return LADE_EINVAL;
  if ((reinterpret_cast<uintptr_t>(logits) | reinterpret_cast<uintptr_t>(out)) % sizeof(T)) return LADE_EINVAL;
  if (ctx->d.D != 1) return LADE_EUNSUPPORTED;    // lookahead parallelism: the accepted n-gram's rows are on one rank
  dim3 grid((vocab + CAP_COLS - 1) / CAP_COLS, ctx->d.GS);
  capture_rows_kernel<T><<<grid, CAP_THREADS, 0, (cudaStream_t)stream>>>(
      ctx->state, ctx->d, (const T*)logits, ld, vocab, ids, lm_rows, meta, result, sampling, (T*)out, ld_out, out_rows);
  LADE_LAUNCH_CHECK("capture_rows_kernel");
  return LADE_OK;
}

}  // namespace lade

using namespace lade;

extern "C" {

int lade_capture_rows(LadeCtx* ctx, void* stream, const void* logits, int32_t ld, int32_t vocab, const int32_t* ids,
                      const int32_t* lm_rows, const int32_t* meta, const int32_t* result, int32_t sampling, void* out,
                      int32_t ld_out, int32_t out_rows) {
  return launch_capture_rows<__nv_bfloat16>(ctx, stream, logits, ld, vocab, ids, lm_rows, meta, result, sampling, out,
                                            ld_out, out_rows);
}

int lade_capture_rows_f16(LadeCtx* ctx, void* stream, const void* logits, int32_t ld, int32_t vocab, const int32_t* ids,
                          const int32_t* lm_rows, const int32_t* meta, const int32_t* result, int32_t sampling,
                          void* out, int32_t ld_out, int32_t out_rows) {
  return launch_capture_rows<__half>(ctx, stream, logits, ld, vocab, ids, lm_rows, meta, result, sampling, out, ld_out,
                                     out_rows);
}

}  // extern "C"
