// Hopper (sm_90a) PTX wrappers shared by the tensor-core kernels: mbarrier, TMA, wgmma, cluster / DSMEM.
#pragma once
#include "common.cuh"

#include <cuda.h>
#include <type_traits>

namespace lade {

// ---- PTX wrappers -------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must trap (launch failure) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}

// ---- wgmma (warpgroup MMA, sm_90a) ------------------------------------------------------------------------
// Shared-memory matrix descriptor, SWIZZLE_128B (cute::GMMA::GmmaDescriptor):
//   bits [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [62,64) layout = 1 (128-byte swizzle)
// K-major operands: SBO = 1024 (next 8 rows), LBO unused.  MN-major operands: LBO = next 64-element block along M/N,
// SBO = next 8 rows along K.
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int N>
__device__ __forceinline__ void wg_fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define LADE_WG_O4(d, i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define LADE_WG_O16(d, i) LADE_WG_O4(d, i), LADE_WG_O4(d, i + 4), LADE_WG_O4(d, i + 8), LADE_WG_O4(d, i + 12)
#define LADE_WG_O64(d) LADE_WG_O16(d, 0), LADE_WG_O16(d, 16), LADE_WG_O16(d, 32), LADE_WG_O16(d, 48)
#define LADE_WG_R64 \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, " \
  "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, " \
  "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"

// D[64 x 128] (+)= A[64 x 16] . B[16 x 128]; A and B from shared memory, both K-major; fp32 accumulators.
template <typename ET>
__device__ __forceinline__ void wgmma_m64n128_ss(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (std::is_same<ET, __half>::value) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " LADE_WG_R64 ", %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : LADE_WG_O64(d) : "l"(da), "l"(db), "r"(accumulate));
  } else {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " LADE_WG_R64 ", %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : LADE_WG_O64(d) : "l"(da), "l"(db), "r"(accumulate));
  }
}
// D[64 x 128] += A[64 x 16] . B[16 x 128]; A from registers (the m64k16 fragment: 4 packed pairs per thread), B from
// shared memory, MN-major (transposed).
template <typename ET>
__device__ __forceinline__ void wgmma_m64n128_rs_tb(float (&d)[64], const uint32_t* a, uint64_t db) {
  if constexpr (std::is_same<ET, __half>::value) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " LADE_WG_R64 ", {%64, %65, %66, %67}, %68, 1, 1, 1, 1;"
                 : LADE_WG_O64(d) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
  } else {
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " LADE_WG_R64 ", {%64, %65, %66, %67}, %68, 1, 1, 1, 1;"
                 : LADE_WG_O64(d) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
  }
}
// D[64 x 32] += A[64 x 16] . B[16 x 32], bf16, both K-major from shared memory.
__device__ __forceinline__ void wgmma_m64n32_ss_bf16(float (&d)[16], uint64_t da, uint64_t db) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, 1, 1, 1, 0, 0;"
               : LADE_WG_O16(d, 0) : "l"(da), "l"(db));
}

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ void named_bar_sync(int id, int n_threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n_threads) : "memory");
}
// The reference's two rounding points of a score pair: r = T(T(s) * c), returned as fp32 (T = the model dtype).
// bf16: the halves of a packed pair are unpacked by hand with one shift and one mask; fp16 needs real conversions.
template <typename ET>
__device__ __forceinline__ void round_scale_round2(float a, float b, float c, float& r0, float& r1);
template <>
__device__ __forceinline__ void round_scale_round2<__nv_bfloat16>(float a, float b, float c, float& r0, float& r1) {
  __nv_bfloat162 v1 = __floats2bfloat162_rn(a, b);
  const uint32_t u1 = *reinterpret_cast<uint32_t*>(&v1);
  __nv_bfloat162 v2 = __floats2bfloat162_rn(__uint_as_float(u1 << 16) * c, __uint_as_float(u1 & 0xffff0000u) * c);
  const uint32_t u2 = *reinterpret_cast<uint32_t*>(&v2);
  r0 = __uint_as_float(u2 << 16);
  r1 = __uint_as_float(u2 & 0xffff0000u);
}
template <>
__device__ __forceinline__ void round_scale_round2<__half>(float a, float b, float c, float& r0, float& r1) {
  const float2 f1 = __half22float2(__floats2half2_rn(a, b));
  const float2 f2 = __half22float2(__floats2half2_rn(f1.x * c, f1.y * c));
  r0 = f2.x;
  r1 = f2.y;
}

__device__ __forceinline__ unsigned pack2_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<unsigned*>(&v);
}

// Programmatic dependent launch (no-ops when the grid was launched without the attribute / has no dependents).
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ uint32_t dsmem_addr(uint32_t local_smem_addr, uint32_t cta_rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(cta_rank));
  return r;
}
__device__ __forceinline__ float4 ld_dsmem_f4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
// coherent (L2) loads of data written by other SMs during this kernel: never the read-only / L1-allocating path
__device__ __forceinline__ float4 ld_global_f4(const float* p) {
  float4 v;
  asm volatile("ld.global.cg.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ float2 ld_global_f2(const float2* p) {
  float2 v;
  asm volatile("ld.global.cg.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p));
  return v;
}


// cuTensorMapEncodeTiled resolved through cudaGetDriverEntryPoint (no libcuda link dependency); null if unavailable.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode_fn();

}  // namespace lade
