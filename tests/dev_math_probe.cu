// TEST INFRASTRUCTURE: the product's math primitives, run over an argument array on the device AND on the host, so that
// tests/test_device_math_gpu.py can compare both with mpmath and with each other.  The product headers are included
// unchanged; the device half is compiled with the library's nvcc flags (default FMA contraction, as the kernels see
// it), the host half with -ffp-contract=off (as the oracle and the tests' host builds).
//   sbm_det_exp / sbm_det_log          include/sb_detmath.h
//   sb::fast_rcp / exp_digamma_shifted salmon_b200/csrc/em_math.h
//   sb::digamma_pos                    salmon_b200/csrc/common.cuh (device only)
//   sbmap::log_add / quant40           salmon_b200/csrc/map_core.h
#include <stdint.h>
#include <string.h>

#include <cuda_runtime.h>

#include "../salmon_b200/csrc/common.cuh"
#include "../salmon_b200/csrc/em_math.h"
#include "../salmon_b200/csrc/map_core.h"

enum Op { OP_EXP = 0, OP_LOG = 1, OP_RCP = 2, OP_EXP_DIGAMMA = 3, OP_DIGAMMA = 4, OP_LOG_ADD = 5, OP_QUANT40 = 6 };

// one result as 64 raw bits (quant40 returns an integer)
__host__ __device__ static uint64_t apply(int op, double a, double b, bool* have) {
  double r = 0.0;
  *have = true;
  switch (op) {
    case OP_EXP: r = sbm_det_exp(a); break;
    case OP_LOG: r = sbm_det_log(a); break;
    case OP_RCP: r = sb::fast_rcp(a); break;
    case OP_EXP_DIGAMMA: r = sb::exp_digamma_shifted(a, b); break;
    case OP_DIGAMMA:
#if defined(__CUDA_ARCH__)
      r = sb::digamma_pos(a);
#else
      *have = false;   // device-only function
#endif
      break;
    case OP_LOG_ADD: r = sbmap::log_add(a, b); break;
    case OP_QUANT40: { const long long q = sbmap::quant40(a); uint64_t u; memcpy(&u, &q, 8); return u; }
    default: *have = false;
  }
  uint64_t u;
  memcpy(&u, &r, 8);
  return u;
}

__global__ void k_probe(int op, uint64_t n, const double* a, const double* b, uint64_t* out) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    bool have;
    out[i] = apply(op, a[i], b[i], &have);
  }
}

// dev_out / host_out: n raw 64-bit results (host_out untouched where the op has no host form).  Returns 0, or a CUDA
// error code, or -1 for an unknown op / no host form when host_out is given.
extern "C" int dmp_run(int op, uint64_t n, const double* a, const double* b, uint64_t* dev_out, uint64_t* host_out) {
  if (op < OP_EXP || op > OP_QUANT40) return -1;
  if (host_out) {
    for (uint64_t i = 0; i < n; ++i) {
      bool have;
      const uint64_t v = apply(op, a[i], b[i], &have);
      if (!have) return -1;
      host_out[i] = v;
    }
  }
  if (!dev_out || n == 0) return 0;
  double *da = nullptr, *db = nullptr;
  uint64_t* dout = nullptr;
  cudaError_t e = cudaMalloc(&da, n * 8);
  if (e == cudaSuccess) e = cudaMalloc(&db, n * 8);
  if (e == cudaSuccess) e = cudaMalloc(&dout, n * 8);
  if (e == cudaSuccess) e = cudaMemcpy(da, a, n * 8, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(db, b, n * 8, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    const uint64_t blocks = (n + 255) / 256;
    k_probe<<<(unsigned)(blocks < 4096 ? blocks : 4096), 256>>>(op, n, da, db, dout);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpy(dev_out, dout, n * 8, cudaMemcpyDeviceToHost);
  cudaFree(da);
  cudaFree(db);
  cudaFree(dout);
  return (int)e;
}
