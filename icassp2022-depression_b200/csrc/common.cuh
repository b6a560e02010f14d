// common.cuh — shared device/host helpers for the b200rnn sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/b200rnn.h"

namespace b200rnn {

// ---- error plumbing (thread-local message, int codes across the C ABI) -------------------------
void set_error(const char* fmt, ...);
void count_launch(int n = 1);  // bumps the counter behind b200rnn_launch_count()
#define B200_CUDA_CHECK(expr)                                                                      \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      ::b200rnn::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__,       \
                           __LINE__);                                                              \
      return B200RNN_ERR_CUDA;                                                                     \
    }                                                                                              \
  } while (0)

// ---- per-device state ----------------------------------------------------------------------------
// cudaFuncSetAttribute and the occupancy queries are per device: every "done once" cache of the launchers is keyed by
// the CURRENT device ordinal, so a process that drives several GPUs (or a module living on cuda:1 while cuda:0 is the
// process default) sets the attributes on each of them. The Python bridge makes the tensor's device current first.
constexpr int MAX_DEVICES = 64;
// SMs of an H100 SXM: sizes the grid-stride launches (one or a few waves) and fixed-order partial-sum buffers
constexpr int NUM_SMS = 132;
inline int current_device() {
  int d = 0;
  if (cudaGetDevice(&d) != cudaSuccess) {
    cudaGetLastError();
    d = 0;
  }
  return (d < 0 || d >= MAX_DEVICES) ? 0 : d;
}

// ---- two-level row addressing ------------------------------------------------------------------
// A logical row index r = outer*inner_n + inner maps to element offset
//   outer*s_outer + inner*s_inner.
// This is how one kernel consumes time-major [T,B,*], batch_first [B,T,*] and permuted views alike.
struct RowMap {
  long long s_outer;
  long long s_inner;
  int inner_n;  // >= 1
  __host__ __device__ __forceinline__ long long off(int r) const {
    int o = r / inner_n;
    int i = r - o * inner_n;
    return (long long)o * s_outer + (long long)i * s_inner;
  }
};
static inline RowMap simple_rows(long long ld) { return RowMap{0, ld, 0x7fffffff}; }
// rows indexed r = t*B + b, memory at t*s_t + b*s_b
static inline RowMap tb_rows(long long s_t, long long s_b, int B) { return RowMap{s_t, s_b, B}; }

// ---- Philox4x32-10 (counter-based RNG for the inter-layer dropout mask) --------------------------
struct Philox4 {
  uint32_t x, y, z, w;
};
__host__ __device__ __forceinline__ void philox_mulhilo(uint32_t a, uint32_t b, uint32_t& hi, uint32_t& lo) {
#ifdef __CUDA_ARCH__
  hi = __umulhi(a, b);
  lo = a * b;
#else
  unsigned long long p = (unsigned long long)a * b;
  hi = (uint32_t)(p >> 32);
  lo = (uint32_t)p;
#endif
}
__host__ __device__ __forceinline__ Philox4 philox4x32_10(uint64_t seed, uint64_t ctr_lo, uint64_t ctr_hi) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  uint32_t c0 = (uint32_t)ctr_lo, c1 = (uint32_t)(ctr_lo >> 32), c2 = (uint32_t)ctr_hi,
           c3 = (uint32_t)(ctr_hi >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0, lo0, hi1, lo1;
    philox_mulhilo(0xD2511F53u, c0, hi0, lo0);
    philox_mulhilo(0xCD9E8D57u, c2, hi1, lo1);
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return Philox4{c0, c1, c2, c3};
}

// ---- activations ------------------------------------------------------------------------------------
// The gate math sits on the serial critical path of every time step, so it uses the hardware ex2 / rcp
// approximations (abs error ~1e-7, two orders below the 1e-5 parity budget) instead of libm expf / tanhf.
__device__ __forceinline__ float sigmoid_f(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ float tanh_f(float x) { return 1.0f - __fdividef(2.0f, 1.0f + __expf(2.0f * x)); }

}  // namespace b200rnn
