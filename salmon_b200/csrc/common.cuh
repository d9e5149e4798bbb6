// common.cuh -- shared helpers for libsalmon_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#include "../../include/salmon_b200.h"

namespace sb {

void set_error(const char* fmt, ...);

#define SB_CUDA(call)                                                          \
  do {                                                                         \
    cudaError_t _e = (call);                                                   \
    if (_e != cudaSuccess) {                                                   \
      sb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call,              \
                    cudaGetErrorString(_e));                                   \
      return SB_ERR_CUDA;                                                      \
    }                                                                          \
  } while (0)

#ifndef SB_TRY
#define SB_TRY(x) do { int _r = (x); if (_r != SB_OK) return _r; } while (0)
#endif

// ---- PTX wrappers: mbarrier + 1-D bulk (TMA) copies ------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_global() {
  asm volatile("fence.proxy.async.global;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// cp.async.bulk global -> shared, completion on an mbarrier (SASS: UBLKCP).
// dst/src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// L2 eviction-priority policies for the bulk copies (createpolicy + .L2::cache_hint)
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void bulk_g2s_hint(void* smem_dst, const void* gsrc, uint32_t bytes,
                                              uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint "
      "[%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}

// ---- warp / block reductions (fixed order => deterministic) -----------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// All threads of the block must call.  scratch: >= 32 doubles of shared memory.
// Result valid in every thread.
template <bool IS_MAX>
__device__ __forceinline__ double block_reduce(double v, double* scratch) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int nw = (blockDim.x + 31) >> 5;
  v = IS_MAX ? warp_max(v) : warp_sum(v);
  __syncthreads();
  if (lane == 0) scratch[wid] = v;
  __syncthreads();
  double r = (lane < nw) ? scratch[lane] : (IS_MAX ? -1.0 : 0.0);
  r = IS_MAX ? warp_max(r) : warp_sum(r);
  return r;
}

// ---- digamma (f64) ----------------------------------------------------------
// Same published Boost.Math 53-bit algorithm the oracle restates
// (reference call sites: src/inference/CollapsedEMOptimizer.cpp:119,127,256,269).
__device__ __forceinline__ double digamma_large(double x) {
  x -= 1.0;
  double result = log(x);
  result += 1.0 / (2.0 * x);
  const double z = 1.0 / (x * x);
  double p = -0.44325980392156862745098039215686274509803921568627;
  p = p * z + 0.083333333333333333333333333333333333333333333333333;
  p = p * z + -0.021092796092796092796092796092796092796092796092796;
  p = p * z + 0.0075757575757575757575757575757575757575757575757576;
  p = p * z + -0.0041666666666666666666666666666666666666666666666667;
  p = p * z + 0.003968253968253968253968253968253968253968253968254;
  p = p * z + -0.0083333333333333333333333333333333333333333333333333;
  p = p * z + 0.083333333333333333333333333333333333333333333333333;
  return result - z * p;
}
__device__ __forceinline__ double digamma_1_2(double x) {
  const double Y = 0.99558162689208984;  // float constant, exactly representable
  const double root1 = 1569415565.0 / 1073741824.0;
  const double root2 = (381566830.0 / 1073741824.0) / 1073741824.0;
  const double root3 = 0.9016312093258695918615325266959189453125e-19;
  double g = x - root1;
  g -= root2;
  g -= root3;
  const double z = x - 1.0;
  double p = -0.0020713321167745952;
  p = p * z + -0.045251321448739056;
  p = p * z + -0.28919126444774784;
  p = p * z + -0.65031853770896507;
  p = p * z + -0.32555031186804491;
  p = p * z + 0.25479851061131551;
  double q = -0.55789841321675513e-6;
  q = q * z + 0.0021284987017821144;
  q = q * z + 0.054151797245674225;
  q = q * z + 0.43593529692665969;
  q = q * z + 1.4606242909763515;
  q = q * z + 2.0767117023730469;
  q = q * z + 1.0;
  const double r = p / q;
  return g * Y + g * r;
}
// x > 0 only (callers guard with digammaMin = 1e-10).
__device__ __forceinline__ double digamma_pos(double x) {
  if (x >= 10.0) return digamma_large(x);
  double result = 0.0;
  while (x > 2.0) {
    x -= 1.0;
    result += 1.0 / x;
  }
  while (x < 1.0) {
    result -= 1.0 / x;
    x += 1.0;
  }
  return result + digamma_1_2(x);
}

}  // namespace sb
