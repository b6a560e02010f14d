// h16.cu — the conversions of the 16-bit modules (h16.cuh): exact widening of what the fp32 kernels read, one
// round-to-nearest-even narrowing of every output. Element-wise and HBM-bound.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <string.h>

#include "h16.cuh"

namespace b200rnn {

namespace {

__device__ __forceinline__ float widen(uint16_t v, int dt) {
  return dt == DT_BF16 ? __uint_as_float((uint32_t)v << 16) : __half2float(__ushort_as_half(v));
}
__device__ __forceinline__ uint16_t narrow(float v, int dt) {
  return dt == DT_BF16 ? __bfloat16_as_ushort(__float2bfloat16_rn(v)) : __half_as_ushort(__float2half_rn(v));
}

// Rows are walked by blocks and columns by threads (no per-element division). When both sides are dense and 8-byte /
// 16-byte aligned (the parameters, states and gradients) the whole range is one row of 4-element vectors.
__global__ void widen16_kernel(const uint16_t* __restrict__ src, RowMap rows, int R, int C, int dt,
                               float* __restrict__ dst, int vec) {
  if (vec) {
    const size_t n4 = (size_t)R * C / 4;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
      const ushort4 v = reinterpret_cast<const ushort4*>(src)[i];
      reinterpret_cast<float4*>(dst)[i] = make_float4(widen(v.x, dt), widen(v.y, dt), widen(v.z, dt), widen(v.w, dt));
    }
    return;
  }
  for (int r = blockIdx.x; r < R; r += gridDim.x) {
    const uint16_t* s = src + rows.off(r);
    float* d = dst + (size_t)r * C;
    for (int c = threadIdx.x; c < C; c += blockDim.x) d[c] = widen(s[c], dt);
  }
}

__global__ void narrow16_kernel(const float* __restrict__ src, RowMap src_rows, int R, int C, int dt,
                                uint16_t* __restrict__ dst, RowMap dst_rows, int accumulate, float* __restrict__ wb,
                                int vec) {
  if (vec) {
    const size_t n4 = (size_t)R * C / 4;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
      float4 v = reinterpret_cast<const float4*>(src)[i];
      ushort4* d = reinterpret_cast<ushort4*>(dst) + i;
      if (accumulate) {
        const ushort4 o = *d;
        v.x += widen(o.x, dt); v.y += widen(o.y, dt); v.z += widen(o.z, dt); v.w += widen(o.w, dt);
      }
      const ushort4 o = make_ushort4(narrow(v.x, dt), narrow(v.y, dt), narrow(v.z, dt), narrow(v.w, dt));
      *d = o;
      if (wb)
        reinterpret_cast<float4*>(wb)[i] = make_float4(widen(o.x, dt), widen(o.y, dt), widen(o.z, dt), widen(o.w, dt));
    }
    return;
  }
  for (int r = blockIdx.x; r < R; r += gridDim.x) {
    const float* s = src + src_rows.off(r);
    uint16_t* d = dst + dst_rows.off(r);
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      float v = s[c];
      if (accumulate) v += widen(d[c], dt);
      const uint16_t o = narrow(v, dt);
      d[c] = o;
      if (wb) wb[(size_t)r * C + c] = widen(o, dt);
    }
  }
}

__global__ void copy16_kernel(const uint16_t* __restrict__ src, RowMap rows, int R, int C, uint16_t* __restrict__ dst) {
  for (int r = blockIdx.x; r < R; r += gridDim.x) {
    const uint16_t* s = src + rows.off(r);
    for (int c = threadIdx.x; c < C; c += blockDim.x) dst[(size_t)r * C + c] = s[c];
  }
}

// The segments of one launch_round16_multi call: each takes ceil(n / ROUND16_CHUNK) consecutive blocks from blk0[s]
constexpr int ROUND16_CHUNK = 4096;
struct Round16Table {
  Round16Seg seg[ROUND16_MAX_SEGS];
  int blk0[ROUND16_MAX_SEGS + 1];
  int nseg;
};

__global__ void __launch_bounds__(256) round16_multi_kernel(const __grid_constant__ Round16Table t, int dt, int mode) {
  int s = 0;
  while (s + 1 < t.nseg && (int)blockIdx.x >= t.blk0[s + 1]) ++s;
  const float* src = t.seg[s].src;
  uint16_t* d16 = t.seg[s].d16;
  float* d32 = t.seg[s].d32;
  const long long base = (long long)(blockIdx.x - t.blk0[s]) * ROUND16_CHUNK;
  const long long n = t.seg[s].n - base < ROUND16_CHUNK ? t.seg[s].n - base : ROUND16_CHUNK;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const long long j = base + i;
    const uint16_t r = narrow(src[j], dt);
    const float w = widen(r, dt);
    if (d16) d16[j] = r;
    if (d32) d32[j] = mode == ROUND16_GRAD_ADD ? d32[j] + w : w;
  }
}

// dense rows (row r at r * C) on both sides, whole 4-element vectors, aligned for them
bool dense_vec(const RowMap& a, const RowMap& b, int R, int C, const void* p16, const void* p32, const void* wb) {
  auto dense = [&](const RowMap& m) { return R == 1 || (m.s_inner == C && (m.inner_n >= R || m.s_outer == (long long)m.inner_n * C)); };
  const uintptr_t al = reinterpret_cast<uintptr_t>(p16) % 8 | reinterpret_cast<uintptr_t>(p32) % 16 |
                       reinterpret_cast<uintptr_t>(wb) % 16;
  return dense(a) && dense(b) && ((size_t)R * C) % 4 == 0 && al == 0;
}

int rows_blocks(int R) { return R < NUM_SMS * 16 ? (R < 1 ? 1 : R) : NUM_SMS * 16; }

int blocks_for(size_t n) {
  size_t b = (n + 255) / 256;
  if (b > (size_t)NUM_SMS * 16) b = (size_t)NUM_SMS * 16;
  return b < 1 ? 1 : (int)b;
}

}  // namespace

int launch_widen16(const void* src, const RowMap& rows, int R, int C, int dt, float* dst, cudaStream_t stream) {
  if ((size_t)R * C == 0) return B200RNN_OK;
  const bool vec = dense_vec(rows, simple_rows(C), R, C, src, dst, nullptr);
  widen16_kernel<<<vec ? blocks_for((size_t)R * C / 4) : rows_blocks(R), 256, 0, stream>>>(
      static_cast<const uint16_t*>(src), rows, R, C, dt, dst, vec ? 1 : 0);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

int launch_narrow16(const float* src, const RowMap& src_rows, int R, int C, int dt, void* dst, const RowMap& dst_rows,
                    bool accumulate, float* wb, cudaStream_t stream) {
  if ((size_t)R * C == 0) return B200RNN_OK;
  const bool vec = dense_vec(dst_rows, src_rows, R, C, dst, src, wb);
  narrow16_kernel<<<vec ? blocks_for((size_t)R * C / 4) : rows_blocks(R), 256, 0, stream>>>(
      src, src_rows, R, C, dt, static_cast<uint16_t*>(dst), dst_rows, accumulate ? 1 : 0, wb, vec ? 1 : 0);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

int launch_round16_multi(const Round16Seg* segs, int nseg, int dt, int mode, cudaStream_t stream) {
  if (nseg > ROUND16_MAX_SEGS) {
    set_error("round16: %d parameter tensors, at most %d", nseg, ROUND16_MAX_SEGS);
    return B200RNN_ERR_UNSUPPORTED;
  }
  Round16Table t;
  memset(&t, 0, sizeof(t));
  long long blocks = 0;
  for (int s = 0; s < nseg; ++s) {  // empty segments (a gradient not asked for) take no block
    if (segs[s].n <= 0 || (!segs[s].d16 && !segs[s].d32)) continue;
    t.seg[t.nseg] = segs[s];
    t.blk0[t.nseg++] = (int)blocks;
    blocks += (segs[s].n + ROUND16_CHUNK - 1) / ROUND16_CHUNK;
  }
  t.blk0[t.nseg] = (int)blocks;
  if (blocks == 0) return B200RNN_OK;
  round16_multi_kernel<<<(unsigned)blocks, 256, 0, stream>>>(t, dt, mode);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

int launch_copy16(const void* src, const RowMap& rows, int R, int C, void* dst, cudaStream_t stream) {
  if ((size_t)R * C == 0) return B200RNN_OK;
  copy16_kernel<<<rows_blocks(R), 256, 0, stream>>>(static_cast<const uint16_t*>(src), rows, R, C,
                                                               static_cast<uint16_t*>(dst));
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

}  // namespace b200rnn
