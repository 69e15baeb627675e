// Memory-bound glue kernels of the decoder layer, with the reference's bf16 rounding points.
//   RMSNorm (+ fused residual add)   lade/models/modeling_llama.py:222-227, :883-889
//   rotary embedding + KV append     lade/models/modeling_llama.py:342-346, :513-516
//   SwiGLU                            lade/models/modeling_llama.py:378
// All are HBM-bound byte movers: 16-byte vectorised, coalesced, one pass over the data.
#include "common.cuh"

#include <cstdlib>

namespace lade {

// Programmatic dependent launch on the glue kernels: every kernel orders itself behind its stream predecessor with
// griddepcontrol.wait as its first instruction (so it is correct whatever the predecessor does) and then lets ITS
// dependent start launching at once.  Whether a neighbouring library GEMM takes part is up to the library (a kernel
// launched without the attribute, or one that never triggers, simply behaves like a normal stream-ordered launch).
__device__ __forceinline__ void pdl_enter() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

static bool pdl_glue_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("LADE_PDL_GLUE");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v != 0;
}

// kernel launch with cudaLaunchAttributeProgrammaticStreamSerialization (when enabled)
template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_glue_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One CTA per row.  h = bf16(x + delta) (if delta), out = w * bf16(h_f32 * rsqrt(mean(h^2) + eps)).
template <bool GATHER, typename T>
__global__ void __launch_bounds__(1024) rmsnorm_kernel(const T* __restrict__ x,
                                                      const T* __restrict__ delta,
                                                      const T* __restrict__ w,
                                                      const int* __restrict__ rows_idx,
                                                      T* __restrict__ h_out,
                                                      T* __restrict__ out, int hidden, float eps) {
  extern __shared__ float s_row[];  // hidden floats
  __shared__ float s_part[32];
  pdl_enter();
  const int out_row = blockIdx.x;
  const int in_row = GATHER ? rows_idx[out_row] : out_row;
  const T* xr = x + (long long)in_row * hidden;
  const T* dr = delta ? delta + (long long)in_row * hidden : nullptr;
  const int nvec = hidden / 8;
  float ss = 0.f;
  for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
    uint4 v = reinterpret_cast<const uint4*>(xr)[i];
    T* e = reinterpret_cast<T*>(&v);
    float f[8];
    if (dr) {
      uint4 dv = reinterpret_cast<const uint4*>(dr)[i];
      const T* de = reinterpret_cast<const T*>(&dv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        e[j] = Elem<T>::from_f(Elem<T>::to_f(e[j]) + Elem<T>::to_f(de[j]));   // residual add in the model dtype
        f[j] = Elem<T>::to_f(e[j]);
      }
      if (h_out && !GATHER) reinterpret_cast<uint4*>(h_out + (long long)out_row * hidden)[i] = v;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = Elem<T>::to_f(e[j]);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s_row[i * 8 + j] = f[j];
      ss += f[j] * f[j];
    }
  }
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
  for (int k = 0; k < (int)(blockDim.x >> 5); ++k) tot += s_part[k];
  const float rstd = rsqrtf(tot / (float)hidden + eps);
  T* orow = out + (long long)out_row * hidden;
  for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
    uint4 wv = reinterpret_cast<const uint4*>(w)[i];
    const T* we = reinterpret_cast<const T*>(&wv);
    uint4 ov;
    T* oe = reinterpret_cast<T*>(&ov);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float n = round_to<T>(s_row[i * 8 + j] * rstd);                // .to(input_dtype)
      oe[j] = Elem<T>::from_f(Elem<T>::to_f(we[j]) * n);                   // weight * hidden (model-dtype mul)
    }
    reinterpret_cast<uint4*>(orow)[i] = ov;
  }
}

// RoPE + append.  grid: rows ; block: 256 threads.  Work item = (head, 8-wide slice of the first half):
// the thread rotates elements [8i, 8i+8) of the first half against the same slice of the second half,
// all accesses 16 bytes.  (Hq + 2 Hkv) * D/16 items per row.
template <typename T>
__global__ void __launch_bounds__(1024) rope_append_kernel(
    const T* __restrict__ qkv, const T* __restrict__ cos_tab,
    const T* __restrict__ sin_tab, const int* __restrict__ pos, const int* __restrict__ meta,
    T* __restrict__ q_out, T* __restrict__ k_cache, T* __restrict__ v_cache,
    int q_pad, int n_heads, int n_kv_heads, int D, int kv_capacity, int max_pos) {
  // programmatic dependent launch: let the consumer (lade_attn_fwd) start its prologue and prefetch the cache tiles of
  // earlier steps while this grid runs; it orders itself with griddepcontrol.wait before touching what is written here
  pdl_enter();
  const int r = blockIdx.x;
  const int half = D >> 1;
  const int per_head = half >> 3;                        // 16-byte slices per half head
  const int n_items = (n_heads + 2 * n_kv_heads) * per_head;
  const int ld = (n_heads + 2 * n_kv_heads) * D;
  const int kv_len = meta[LADE_M_KV_LEN];
  const int cache_row = kv_len + r;
  int p = pos[r];
  p = p < 0 ? 0 : (p >= max_pos ? max_pos - 1 : p);
  const T* crow = cos_tab + (long long)p * D;
  const T* srow = sin_tab + (long long)p * D;
  for (int it = threadIdx.x; it < n_items; it += blockDim.x) {
    const int h = it / per_head, sl = it % per_head;
    const T* src = qkv + (long long)r * ld + (long long)h * D + sl * 8;
    const uint4 a = *reinterpret_cast<const uint4*>(src);
    const uint4 b = *reinterpret_cast<const uint4*>(src + half);
    T* dst;
    if (h < n_heads) {
      dst = q_out + ((long long)h * q_pad + r) * D + sl * 8;
    } else if (h < n_heads + n_kv_heads) {
      if (cache_row >= kv_capacity) continue;
      dst = k_cache + ((long long)(h - n_heads) * kv_capacity + cache_row) * D + sl * 8;
    } else {                                              // V: plain append
      if (cache_row >= kv_capacity) continue;
      dst = v_cache + ((long long)(h - n_heads - n_kv_heads) * kv_capacity + cache_row) * D + sl * 8;
      *reinterpret_cast<uint4*>(dst) = a;
      *reinterpret_cast<uint4*>(dst + half) = b;
      continue;
    }
    const uint4 c1 = *reinterpret_cast<const uint4*>(crow + sl * 8);
    const uint4 c2 = *reinterpret_cast<const uint4*>(crow + half + sl * 8);
    const uint4 s1 = *reinterpret_cast<const uint4*>(srow + sl * 8);
    const uint4 s2 = *reinterpret_cast<const uint4*>(srow + half + sl * 8);
    const T* x1 = reinterpret_cast<const T*>(&a);
    const T* x2 = reinterpret_cast<const T*>(&b);
    const T* pc1 = reinterpret_cast<const T*>(&c1);
    const T* pc2 = reinterpret_cast<const T*>(&c2);
    const T* ps1 = reinterpret_cast<const T*>(&s1);
    const T* ps2 = reinterpret_cast<const T*>(&s2);
    uint4 o1v, o2v;
    T* o1 = reinterpret_cast<T*>(&o1v);
    T* o2 = reinterpret_cast<T*>(&o2v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float f1 = Elem<T>::to_f(x1[j]), f2 = Elem<T>::to_f(x2[j]);
      // (q * cos) + (rotate_half(q) * sin), every op rounded to bf16 (modeling_llama.py:344-345)
      o1[j] = Elem<T>::from_f(round_to<T>(f1 * Elem<T>::to_f(pc1[j])) + round_to<T>(-f2 * Elem<T>::to_f(ps1[j])));
      o2[j] = Elem<T>::from_f(round_to<T>(f2 * Elem<T>::to_f(pc2[j])) + round_to<T>(f1 * Elem<T>::to_f(ps2[j])));
    }
    *reinterpret_cast<uint4*>(dst) = o1v;
    *reinterpret_cast<uint4*>(dst + half) = o2v;
  }
}

template <typename T>
__global__ void swiglu_kernel(const T* __restrict__ gate_up, T* __restrict__ out,
                              int rows, int inter) {
  pdl_enter();
  const int nvec = inter / 8;
  const long long total = (long long)rows * nvec;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / nvec), c = (int)(i % nvec);
    const uint4 gv = reinterpret_cast<const uint4*>(gate_up + (long long)r * 2 * inter)[c];
    const uint4 uv = reinterpret_cast<const uint4*>(gate_up + (long long)r * 2 * inter + inter)[c];
    const T* g = reinterpret_cast<const T*>(&gv);
    const T* u = reinterpret_cast<const T*>(&uv);
    uint4 ov;
    T* o = reinterpret_cast<T*>(&ov);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float x = Elem<T>::to_f(g[j]);
      const float s = round_to<T>(x / (1.0f + expf(-x)));                   // silu in fp32, model-dtype result
      o[j] = Elem<T>::from_f(s * Elem<T>::to_f(u[j]));
    }
    reinterpret_cast<uint4*>(out + (long long)r * inter)[c] = ov;
  }
}

}  // namespace lade

using namespace lade;

extern "C" {

static int norm_threads(int hidden) {
  int t = ((hidden / 8 + 31) / 32) * 32;
  return t < 128 ? 128 : (t > 1024 ? 1024 : t);
}

}  // extern "C"  (templated implementations below have C++ linkage)

template <typename T>
static int rmsnorm_impl(void* stream, const void* x, const void* delta, const void* weight, void* h_out, void* out,
                        int32_t rows, int32_t hidden, float eps) {
  if (!x || !weight || !out || rows < 1 || hidden < 8 || hidden % 8 != 0) return LADE_EINVAL;
  if (delta && !h_out) return LADE_EINVAL;
  const size_t smem = sizeof(float) * hidden;
  if (smem > 96 * 1024) return LADE_EUNSUPPORTED;
  if (smem > 48 * 1024)
    LADE_CUDA_CHECK(cudaFuncSetAttribute(rmsnorm_kernel<false, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // one 16-byte vector per thread when the row fits (4096 / 8 = 512 threads): a single round of loads per phase
  const int threads = norm_threads(hidden);
  LADE_CUDA_CHECK(launch_pdl(rmsnorm_kernel<false, T>, dim3(rows), dim3(threads), smem, (cudaStream_t)stream,
                             (const T*)x, (const T*)delta, (const T*)weight, (const int*)nullptr, (T*)h_out, (T*)out,
                             hidden, eps));
  return LADE_OK;
}

template <typename T>
static int rmsnorm_gather_impl(void* stream, const void* x, const void* delta, const void* weight, const int32_t* rows_idx,
                               void* out, int32_t n_rows, int32_t hidden, float eps) {
  if (!x || !weight || !out || !rows_idx || n_rows < 1 || hidden < 8 || hidden % 8 != 0) return LADE_EINVAL;
  const size_t smem = sizeof(float) * hidden;
  if (smem > 96 * 1024) return LADE_EUNSUPPORTED;
  if (smem > 48 * 1024)
    LADE_CUDA_CHECK(cudaFuncSetAttribute(rmsnorm_kernel<true, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int threads = norm_threads(hidden);
  LADE_CUDA_CHECK(launch_pdl(rmsnorm_kernel<true, T>, dim3(n_rows), dim3(threads), smem, (cudaStream_t)stream,
                             (const T*)x, (const T*)delta, (const T*)weight, (const int*)rows_idx, (T*)nullptr, (T*)out,
                             hidden, eps));
  return LADE_OK;
}

template <typename T>
static int rope_append_impl(void* stream, const void* qkv, const void* cos_tab, const void* sin_tab, const int32_t* pos,
                            const int32_t* meta, void* q_out, void* k_cache, void* v_cache, int32_t rows, int32_t q_pad,
                            int32_t n_heads, int32_t n_kv_heads, int32_t head_dim, int32_t kv_capacity, int32_t max_pos) {
  if (!qkv || !cos_tab || !sin_tab || !pos || !meta || !q_out || !k_cache || !v_cache) return LADE_EINVAL;
  if (rows < 1 || rows > q_pad || head_dim % 16 != 0 || head_dim > 512 || n_heads < 1 || n_kv_heads < 1) return LADE_EINVAL;
  // one work item (head, 8-wide slice) per thread when they fit: (32 + 2*32) heads * 8 slices = 768 threads at 7B
  int rope_threads = (((n_heads + 2 * n_kv_heads) * (head_dim / 16) + 31) / 32) * 32;
  rope_threads = rope_threads < 128 ? 128 : (rope_threads > 1024 ? 1024 : rope_threads);
  LADE_CUDA_CHECK(launch_pdl(rope_append_kernel<T>, dim3(rows), dim3(rope_threads), 0, (cudaStream_t)stream,
                             (const T*)qkv, (const T*)cos_tab, (const T*)sin_tab, (const int*)pos, (const int*)meta,
                             (T*)q_out, (T*)k_cache, (T*)v_cache, q_pad, n_heads, n_kv_heads, head_dim, kv_capacity,
                             max_pos));
  return LADE_OK;
}

template <typename T>
static int swiglu_impl(void* stream, const void* gate_up, void* out, int32_t rows, int32_t inter) {
  if (!gate_up || !out || rows < 1 || inter < 8 || inter % 8 != 0) return LADE_EINVAL;
  const long long total = (long long)rows * (inter / 8);
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  LADE_CUDA_CHECK(launch_pdl(swiglu_kernel<T>, dim3(blocks), dim3(256), 0, (cudaStream_t)stream,
                             (const T*)gate_up, (T*)out, rows, inter));
  return LADE_OK;
}

extern "C" {

// bf16 models (the BASELINE configs) and, with the _f16 suffix, fp16 models (the dtype of the reference's README /
// minimal.py): same kernels instantiated on the element type, every rounding point in the model dtype
int lade_rmsnorm(void* stream, const void* x, const void* delta, const void* weight, void* h_out, void* out,
                 int32_t rows, int32_t hidden, float eps) {
  return rmsnorm_impl<__nv_bfloat16>(stream, x, delta, weight, h_out, out, rows, hidden, eps);
}
int lade_rmsnorm_f16(void* stream, const void* x, const void* delta, const void* weight, void* h_out, void* out,
                     int32_t rows, int32_t hidden, float eps) {
  return rmsnorm_impl<__half>(stream, x, delta, weight, h_out, out, rows, hidden, eps);
}
int lade_rmsnorm_gather(void* stream, const void* x, const void* delta, const void* weight,
                        const int32_t* rows_idx, void* out, int32_t n_rows, int32_t hidden, float eps) {
  return rmsnorm_gather_impl<__nv_bfloat16>(stream, x, delta, weight, rows_idx, out, n_rows, hidden, eps);
}
int lade_rmsnorm_gather_f16(void* stream, const void* x, const void* delta, const void* weight,
                            const int32_t* rows_idx, void* out, int32_t n_rows, int32_t hidden, float eps) {
  return rmsnorm_gather_impl<__half>(stream, x, delta, weight, rows_idx, out, n_rows, hidden, eps);
}
int lade_rope_append(void* stream, const void* qkv, const void* cos_tab, const void* sin_tab,
                     const int32_t* pos, const int32_t* meta, void* q_out, void* k_cache, void* v_cache,
                     int32_t rows, int32_t q_pad, int32_t n_heads, int32_t n_kv_heads, int32_t head_dim,
                     int32_t kv_capacity, int32_t max_pos) {
  return rope_append_impl<__nv_bfloat16>(stream, qkv, cos_tab, sin_tab, pos, meta, q_out, k_cache, v_cache, rows, q_pad,
                                         n_heads, n_kv_heads, head_dim, kv_capacity, max_pos);
}
int lade_rope_append_f16(void* stream, const void* qkv, const void* cos_tab, const void* sin_tab,
                         const int32_t* pos, const int32_t* meta, void* q_out, void* k_cache, void* v_cache,
                         int32_t rows, int32_t q_pad, int32_t n_heads, int32_t n_kv_heads, int32_t head_dim,
                         int32_t kv_capacity, int32_t max_pos) {
  return rope_append_impl<__half>(stream, qkv, cos_tab, sin_tab, pos, meta, q_out, k_cache, v_cache, rows, q_pad,
                                  n_heads, n_kv_heads, head_dim, kv_capacity, max_pos);
}
int lade_swiglu(void* stream, const void* gate_up, void* out, int32_t rows, int32_t inter) {
  return swiglu_impl<__nv_bfloat16>(stream, gate_up, out, rows, inter);
}
int lade_swiglu_f16(void* stream, const void* gate_up, void* out, int32_t rows, int32_t inter) {
  return swiglu_impl<__half>(stream, gate_up, out, rows, inter);
}

}  // extern "C"
