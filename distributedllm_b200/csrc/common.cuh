// common.cuh -- error plumbing and sm_90a PTX helpers shared by the slice runtime.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>
#include <string>

#include "../../include/b200_slice.h"

namespace b200 {

// ---- thread-local last error (b200_last_error) -------------------------------------------
inline std::string & last_error_ref() { static thread_local std::string e; return e; }
inline int fail(int code, const char * fmt, ...) {
    char buf[1024];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    last_error_ref() = buf;
    return code;
}
#define B200_CUDA(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) \
    return b200::fail(B200_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)

// ---- exact-arithmetic helpers: never let nvcc contract a*b+c on the parity path -------------
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float ffma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ float h2f(uint16_t h) { return __half2float(__ushort_as_half(h)); }
__device__ __forceinline__ uint16_t f2h(float f) { return __half_as_ushort(__float2half_rn(f)); }

// ---- mbarrier / bulk-copy (TMA 1-D) / programmatic dependent launch ------------------------
__device__ __forceinline__ uint32_t smem_u32(const void * p) { return (uint32_t) __cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t * bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t * bar) {
    asm volatile("{ .reg .b64 st; mbarrier.arrive.shared::cta.b64 st, [%0]; }" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t * bar, uint32_t bytes) {
    asm volatile("{ .reg .b64 st; mbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1; }"
                 :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t * bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t * bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) { }
}
// 1-D bulk async copy global -> shared, completion counted on an mbarrier (SASS: UBLKCP).
// Weights are streamed once per token and are far larger than L2: mark them evict-first.
__device__ __forceinline__ void bulk_g2s(void * dst_smem, const void * src_gmem, uint32_t bytes, uint64_t * bar) {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 :: "r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(pol) : "memory");
}
// 1-D bulk async copy shared -> global, tracked by bulk groups: s2g ... s2g, bulk_commit, then bulk_wait_read<N> before the
// shared source is overwritten (at most N newer groups may still be reading) and bulk_wait<0> before the CTA exits.
__device__ __forceinline__ void s2g(void * dst_gmem, const void * src_smem, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 :: "l"(dst_gmem), "r"(smem_u32(src_smem)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" :: "n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" :: "n"(N) : "memory"); }
// 16-byte load that asks L2 to keep the line (evict_last): small, hot, read-every-token data (norm weights) must
// survive the evict_first weight stream, otherwise every token pays an HBM round trip for it under full load
__device__ __forceinline__ float4 ldg_keep(const float * p) {
    uint64_t pol; float4 v;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    asm volatile("ld.global.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ void grid_dep_wait()   { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void grid_dep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
// debug timeline: 8 timestamps per CTA (blockIdx.x + gridDim.x * blockIdx.y)
#define B200_TRACE(ptr, slot) do { if (ptr) (ptr)[((size_t) blockIdx.y * gridDim.x + blockIdx.x) * 8 + (slot)] = b200::gtime(); } while (0)

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(nthreads) : "memory");
}

}  // namespace b200
